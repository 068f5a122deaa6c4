"""Drop-in mirror of the reference's `bruce_slam` package for its sonar front-end hot path.

Same module and function names as jake3991/sonar-SLAM's bruce_slam (native modules
`cfar`, `pcl`; classes `CFAR`, `FeatureExtraction`; scan-matching helpers of `SLAM`),
backed by libsonarfe.so (hand-written CUDA for H100) through ctypes.  To use it under the
reference's own import names put this directory's parent on sys.path:

    import sys, sonar_slam_b200; sys.path.insert(0, sonar_slam_b200.__path__[0])
    from bruce_slam import cfar, pcl
    from bruce_slam.CFAR import CFAR
"""
