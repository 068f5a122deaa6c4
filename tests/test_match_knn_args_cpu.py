"""CPU-only: `bruce_slam.pcl.match_knn` rejects bad arguments before any device work (no GPU needed)."""
import numpy as np
import pytest

from sonar_slam_b200.bruce_slam import pcl


def test_match_knn_rejects_bad_arguments_before_any_device_work():
    ref, q = np.zeros((4, 2), np.float32), np.zeros((3, 2), np.float32)
    with pytest.raises(ValueError, match="knn must be at least 1"):
        pcl.match_knn(ref, q, 0, 0.5)
    with pytest.raises(ValueError, match="knn must be at least 1"):
        pcl.match_knn(ref, q, -3, 0.5)
    with pytest.raises(NotImplementedError, match="at most 16"):
        pcl.match_knn(ref, q, 17, 0.5)
    with pytest.raises(TypeError):
        pcl.match_knn(np.zeros((4, 3), np.float32), q, 2, 0.5)   # 2-column clouds only
    with pytest.raises(TypeError):
        pcl.match_knn(ref, np.zeros(6, np.float32), 2, 0.5)
    ids, d = pcl.match_knn(ref, np.zeros((0, 2), np.float32), 5, 0.5)  # no query: nothing to send to the device
    assert ids.shape == (5, 0) and ids.dtype == np.int32 and d.shape == (5, 0) and d.dtype == np.float32
