"""Wire formats on either side of the front end (SURVEY.md N4), without ROS.

The reference hands the feature cloud from `FeatureExtraction.publish_features` to `SLAMNode.SLAM_callback` as a
`sensor_msgs/PointCloud2` built by `n2r(points, "PointCloudXYZ")` (bruce_slam/utils/conversions.py:276-312 ->
sensor_msgs.point_cloud2.create_cloud_xyz32) and read back with ros_numpy's `pointcloud2_to_xyz_array`
(slam_ros.py:169).  ROS is not part of this image; the classes below carry the same field names and the same bytes
(`data`: little-endian float32 x, y, z per point, point_step 12), so a bag reader or a rospy shim can copy them field by
field, and the sign convention of the hand-off -- (p0, p1) -> [p0, 0, p1] -> (x, -z) -- is exercised end to end.

    n2r(arr, "PointCloudXYZ" | "PointCloudXYZI")      utils/conversions.py:297-308
    r2n(msg)  PointCloud2 -> float64 [width, n_fields]  utils/conversions.py:240-243
              OculusPing  -> gamma-corrected float32   utils/conversions.py:229-235
    pointcloud2_to_xyz_array(msg, remove_nans=True)    ros_numpy.point_cloud2 (slam_ros.py:169)
    feature_msg(ping, points) / keyframe_points(msg)   feature_extraction.py:181-190 / slam_ros.py:169-170
    numpy_to_image(arr, encoding)                      ros_numpy.image (feature_extraction.py:228)
"""
import sys

import numpy as np


class Header(object):
    __slots__ = ("seq", "stamp", "frame_id")

    def __init__(self, seq=0, stamp=None, frame_id=""):
        self.seq, self.stamp, self.frame_id = seq, stamp, frame_id


class PointField(object):
    """sensor_msgs/PointField"""
    INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
    __slots__ = ("name", "offset", "datatype", "count")

    def __init__(self, name="", offset=0, datatype=0, count=1):
        self.name, self.offset, self.datatype, self.count = name, offset, datatype, count


_NP = {PointField.INT8: "i1", PointField.UINT8: "u1", PointField.INT16: "i2", PointField.UINT16: "u2",
       PointField.INT32: "i4", PointField.UINT32: "u4", PointField.FLOAT32: "f4", PointField.FLOAT64: "f8"}


class PointCloud2(object):
    """sensor_msgs/PointCloud2 (same attribute names, `data` = the message's byte string)."""
    _type = "sensor_msgs/PointCloud2"
    __slots__ = ("header", "height", "width", "fields", "is_bigendian", "point_step", "row_step", "data", "is_dense")

    def __init__(self):
        self.header = Header()
        self.height, self.width, self.fields = 1, 0, []
        self.is_bigendian, self.point_step, self.row_step, self.data, self.is_dense = False, 0, 0, b"", False


def create_cloud(header, fields, points):
    """sensor_msgs.point_cloud2.create_cloud: one row, the fields packed in offset order, little endian."""
    points = np.asarray(points)
    n = len(points)
    step = max(f.offset + np.dtype(_NP[f.datatype]).itemsize * f.count for f in fields) if fields else 0
    rec = np.zeros(n, np.dtype({"names": [f.name for f in fields], "formats": ["<" + _NP[f.datatype] for f in fields],
                                "offsets": [f.offset for f in fields], "itemsize": step}))
    cols = points.reshape(n, -1)
    for k, f in enumerate(fields):
        rec[f.name] = cols[:, k]
    msg = PointCloud2()
    msg.header = header
    msg.height, msg.width, msg.fields = 1, n, list(fields)
    msg.is_bigendian, msg.point_step, msg.row_step = False, step, step * n
    msg.data, msg.is_dense = rec.tobytes(), False
    return msg


def _xyz_fields(extra=()):
    f = [PointField("x", 0, PointField.FLOAT32, 1), PointField("y", 4, PointField.FLOAT32, 1),
         PointField("z", 8, PointField.FLOAT32, 1)]
    return f + [PointField(name, 12 + 4 * k, PointField.FLOAT32, 1) for k, name in enumerate(extra)]


def n2r(numpy_arr, msg):
    """numpy -> message (utils/conversions.py:276-312; the point-cloud branches)."""
    if msg == "PointCloudXYZ":
        return create_cloud(Header(), _xyz_fields(), np.array(numpy_arr))        # create_cloud_xyz32
    if msg == "PointCloudXYZI":
        return create_cloud(Header(), _xyz_fields(("i",)), np.array(numpy_arr))
    raise NotImplementedError("Not implemented from numpy array to {}".format(msg))


def _records(msg):
    if msg.is_bigendian:
        raise NotImplementedError("big-endian PointCloud2")
    dt = np.dtype({"names": [f.name for f in msg.fields], "formats": ["<" + _NP[f.datatype] for f in msg.fields],
                   "offsets": [f.offset for f in msg.fields], "itemsize": msg.point_step})
    return np.frombuffer(msg.data, dt, count=msg.width * msg.height)


def r2n(ros_msg):
    """message -> numpy (utils/conversions.py:217-247)."""
    kind = getattr(ros_msg, "_type", None)
    if kind == "sensor_msgs/PointCloud2":
        rec = _records(ros_msg)      # pc2.read_points yields python floats: float64 [width, n_fields]
        cols = sum(f.count for f in ros_msg.fields)
        return np.stack([rec[f.name].astype(np.float64) for f in ros_msg.fields], 1).reshape(ros_msg.width, cols)
    if kind == "sonar_oculus/OculusPing":
        import cv2
        img = np.asarray(ros_msg.ping if isinstance(ros_msg.ping, np.ndarray) else r2n(ros_msg.ping))
        img = np.clip(cv2.pow(img / 255.0, 255.0 / ros_msg.fire_msg.gamma) * 255.0, 0, 255)
        return np.float32(img)
    if kind == "sensor_msgs/Image":
        return np.array(ros_msg.data, "uint8").reshape(ros_msg.height, ros_msg.width, -1).squeeze()
    raise NotImplementedError("Not implemented from {} to numpy".format(str(type(ros_msg))))


def pointcloud2_to_xyz_array(cloud_msg, remove_nans=True):
    """ros_numpy.point_cloud2.pointcloud2_to_xyz_array: float32 [N,3]; rows with a NaN coordinate are dropped."""
    rec = _records(cloud_msg)
    pts = np.stack([rec["x"], rec["y"], rec["z"]], 1).astype(np.float32)
    if remove_nans:
        pts = pts[np.isfinite(pts).all(1)]
    return pts


def feature_msg(ping, points):
    """FeatureExtraction.publish_features (feature_extraction.py:175-193): the in-plane cloud (p0, p1) goes out as
    [p0, 0, p1], stamped like the ping."""
    points = np.asarray(points)
    msg = n2r(np.c_[points[:, 0], np.zeros(len(points)), points[:, 1]], "PointCloudXYZ")
    msg.header.stamp = getattr(getattr(ping, "header", None), "stamp", None)
    msg.header.frame_id = "base_link"
    return msg


def keyframe_points(feature_message):
    """SLAMNode.SLAM_callback (slam_ros.py:169-170): the keyframe's 2-D cloud is (x, -z) of the message."""
    points = pointcloud2_to_xyz_array(feature_message)
    return np.c_[points[:, 0], -1 * points[:, 2]]


class Image(object):
    """sensor_msgs/Image (same attribute names, `data` = the message's byte string)."""
    _type = "sensor_msgs/Image"
    __slots__ = ("header", "height", "width", "encoding", "is_bigendian", "step", "data")

    def __init__(self, encoding=""):
        self.header = Header()
        self.height, self.width, self.encoding, self.is_bigendian, self.step, self.data = 0, 0, encoding, False, 0, b""


# ros_numpy.image.name_to_dtypes: encoding -> (element type, channels)
IMAGE_ENCODINGS = {
    "rgb8": (np.uint8, 3), "rgba8": (np.uint8, 4), "rgb16": (np.uint16, 3), "rgba16": (np.uint16, 4),
    "bgr8": (np.uint8, 3), "bgra8": (np.uint8, 4), "bgr16": (np.uint16, 3), "bgra16": (np.uint16, 4),
    "mono8": (np.uint8, 1), "mono16": (np.uint16, 1),
    "8UC1": (np.uint8, 1), "8UC2": (np.uint8, 2), "8UC3": (np.uint8, 3), "8UC4": (np.uint8, 4),
    "16UC1": (np.uint16, 1), "16UC3": (np.uint16, 3), "32FC1": (np.float32, 1), "32FC3": (np.float32, 3),
}


def numpy_to_image(arr, encoding):
    """ros_numpy.image.numpy_to_image: a sensor_msgs/Image holding `arr` ([height, width] or [height, width,
    channels]) with `encoding`; data is the C-contiguous bytes, step the row stride."""
    if encoding not in IMAGE_ENCODINGS:
        raise TypeError("Unrecognized encoding {}".format(encoding))
    im = Image(encoding=encoding)
    dtype_class, exp_channels = IMAGE_ENCODINGS[encoding]
    if arr.ndim == 2:
        im.height, im.width, channels = arr.shape + (1,)
    elif arr.ndim == 3:
        im.height, im.width, channels = arr.shape
    else:
        raise TypeError("Array must be two or three dimensional")
    if exp_channels != channels:
        raise TypeError("Array has {} channels, {} requires {}".format(channels, encoding, exp_channels))
    if dtype_class != arr.dtype.type:
        raise TypeError("Array is {}, {} requires {}".format(arr.dtype.type, encoding, dtype_class))
    contig = np.ascontiguousarray(arr)
    im.data = contig.tobytes()
    im.step = contig.strides[0]
    im.is_bigendian = arr.dtype.byteorder == ">" or (arr.dtype.byteorder == "=" and sys.byteorder == "big")
    return im
