import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
GOLDEN = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def gpu_ctx():
    """A libsonarfe context on cuda:0.  Fails (not skips) when the library cannot run."""
    import torch
    assert torch.cuda.is_available(), "GPU test selected but no CUDA device is visible"
    from sonar_slam_b200 import ops
    return ops.context(0)


SHIPPED_ICP_YAML = """matcher:
  KDTreeMatcher:
    knn: 1
    epsilon: 0
    maxDist: 10.0
outlierFilters:
  - MaxDistOutlierFilter:
      maxDist: 3.0
  - TrimmedDistOutlierFilter:
      ratio: 0.8
errorMinimizer:
  PointToPointErrorMinimizer
transformationCheckers:
  - CounterTransformationChecker:
      maxIterationCount: 40
  - DifferentialTransformationChecker:
      minDiffRotErr: 0.01
      minDiffTransErr: 0.1
      smoothLength: 4
inspector:
  NullInspector
"""


@pytest.fixture
def icp_yaml(tmp_path):
    """The chain bruce_slam/config/icp.yaml ships (icp.yaml:5-28), as a file ICP.loadFromYaml can read."""
    p = tmp_path / "icp.yaml"
    p.write_text(SHIPPED_ICP_YAML)
    return str(p)
