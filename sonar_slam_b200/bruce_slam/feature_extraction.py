"""`bruce_slam.feature_extraction.FeatureExtraction` -- ROS-free mirror of the reference's node class
(bruce_slam/src/bruce_slam/feature_extraction.py:26-252): same attributes, same method names, same
numeric results; the ROS plumbing (rospy params, subscribers, publishers, cv_bridge) is replaced by
plain arguments and return values.

    fe = FeatureExtraction(); fe.init_node(params_dict_or_feature_yaml); points = fe.callback(ping)

`ping` is any object with the OculusPing fields the reference reads: ping_id, range_resolution,
num_ranges, bearings (int16 centi-degrees) and the image as `image` (uint8 [num_ranges, num_beams]) --
see sonar_slam_b200.synth.Ping.  callback() returns (and keeps in `self.points`) the float32 [K,2]
cloud the reference would publish: column 0 forward range (m), column 1 lateral (m); a skipped ping
gives the same single NaN point the reference publishes (feature_extraction.py:201-207).

The polar->Cartesian maps stay host-side numpy/scipy exactly as in the reference
(generate_map_xy, :134-173, re-run only when the geometry changes); everything per ping runs on the
GPU: CFAR with the amplitude gate fused (:223-224), the remap/nonzero/metres step (:231-238),
pcl.downsample and pcl.remove_outlier (:241-249).  With `render_feature_img` the feature image the reference publishes
(:226-228) is rendered on the GPU too.
"""
import numpy as np
from scipy.interpolate import interp1d

from .. import _lib
from . import pcl
from .CFAR import CFAR

_ALG = {"CA": 0, "SOCA": 1, "GOCA": 2, "OS": 3}


class FeatureExtraction(object):
    """Extract an in-plane 2-D point cloud from polar sonar images with CFAR."""

    def __init__(self):
        # default parameters for CFAR (feature_extraction.py:38-46)
        self.Ntc = 40
        self.Ngc = 10
        self.Pfa = 1e-2
        self.rank = None
        self.alg = "SOCA"
        self.detector = None
        self.threshold = 0
        self.cimg = None

        # default parameters for the point cloud (:48-54)
        self.colormap = "RdBu_r"
        self.pub_rect = True
        self.resolution = 0.5
        self.outlier_filter_radius = 1.0
        self.outlier_filter_min_points = 5
        self.skip = 5

        self.feature_img = None
        # opt-in: also render the bgr8 feature image the reference publishes (:226-228) into `feature_img`, and its
        # sensor_msgs/Image mirror into `feature_img_msg`, on the GPU (sonar_slam_b200.feature_image)
        self.render_feature_img = False
        self.feature_img_msg = None

        # polar -> Cartesian remapping state (:59-70)
        self.res = None
        self.height = None
        self.rows = None
        self.width = None
        self.cols = None
        self.map_x = None
        self.map_y = None
        self.f_bearings = None
        self.to_rad = lambda bearing: bearing * np.pi / 18000
        self.REVERSE_Z = 1
        self.maxRange = None

        self.compressed_images = True
        # opt-in: decode compressed pings that sonar_slam_b200.jpeg or sonar_slam_b200.png accepts on the GPU (same
        # uint8 image bit for bit); other streams (progressive JPEG, palette PNG, ...) keep the cv2 path
        self.decode_on_device = False
        self.rov_id = ""

        # device side
        self._maps = None
        self._maps_shape = None
        self.points = None
        self.locs = None

    def configure(self):
        """Build the CFAR detector object from the current parameters."""
        self.detector = CFAR(self.Ntc, self.Ngc, self.Pfa, self.rank)

    def init_node(self, params=None, ns="~"):
        """`params`: the dict rosparam would hold (the content of config/feature.yaml) or a path to that
        YAML.  Keys as in feature_extraction.py:86-114 (CFAR/{Ntc,Ngc,Pfa,rank,alg},
        filter/{threshold,resolution,radius,min_points,skip}, compressed_images)."""
        if isinstance(params, str):
            import yaml
            with open(params) as f:
                params = yaml.safe_load(f)
        params = params or {}
        cf, fl = params.get("CFAR", {}), params.get("filter", {})
        self.Ntc = cf.get("Ntc", self.Ntc)
        self.Ngc = cf.get("Ngc", self.Ngc)
        self.Pfa = cf.get("Pfa", self.Pfa)
        self.rank = cf.get("rank", self.rank)
        self.alg = cf.get("alg", "SOCA")
        self.threshold = fl.get("threshold", self.threshold)
        self.resolution = fl.get("resolution", self.resolution)
        self.outlier_filter_radius = fl.get("radius", self.outlier_filter_radius)
        self.outlier_filter_min_points = fl.get("min_points", self.outlier_filter_min_points)
        self.skip = fl.get("skip", self.skip)
        self.compressed_images = params.get("compressed_images", False)
        self.configure()

    def generate_map_xy(self, ping):
        """Sampling maps from the Cartesian image back into (range bin, beam) coordinates; cached per
        geometry.  Same expressions as the reference (:142-173)."""
        _res = ping.range_resolution
        _height = ping.num_ranges * _res
        _rows = ping.num_ranges
        _width = np.sin(self.to_rad(ping.bearings[-1] - ping.bearings[0]) / 2) * _height * 2
        _cols = int(np.ceil(_width / _res))
        if self.res == _res and self.height == _height and self.rows == _rows and self.width == _width \
                and self.cols == _cols:
            return
        self.res, self.height, self.rows, self.width, self.cols = _res, _height, _rows, _width, _cols

        bearings = self.to_rad(np.asarray(ping.bearings, dtype=np.float32))
        f_bearings = interp1d(bearings, range(len(bearings)), kind="linear", bounds_error=False, fill_value=-1,
                              assume_sorted=True)
        self.f_bearings = f_bearings
        XX, YY = np.meshgrid(range(self.cols), range(self.rows))
        x = self.res * (self.rows - YY)
        y = self.res * (-self.cols / 2.0 + XX + 0.5)
        b = np.arctan2(y, x) * self.REVERSE_Z
        r = np.sqrt(np.square(x) + np.square(y))
        self.map_y = np.asarray(r / self.res, dtype=np.float32)
        self.map_x = np.asarray(f_bearings(b), dtype=np.float32)
        self._maps = None  # device table is rebuilt on next use

    def device_maps(self, ctx, num_beams):
        """The geometry's sampling table on the GPU (built lazily, cached)."""
        key = (id(ctx), self.rows, self.cols, num_beams, self.width, self.height)
        if self._maps is None or self._maps_shape != key:
            self._maps = _lib.Maps(ctx, self.map_x, self.map_y, self.rows, num_beams, self.width, self.height)
            self._maps_shape = key
        return self._maps

    def publish_features(self, ping, points):
        """The reference publishes a PointCloud2 here (:175-193).  The cloud is kept and returned as before; the
        message itself (same bytes, no ROS: bruce_slam/conversions.py) is left in `self.feature_msg` for a caller
        that forwards it."""
        self.points = points
        from . import conversions
        self.feature_msg = conversions.feature_msg(ping, points)
        return points

    def ping_image(self, sonar_msg):
        """The polar uint8 image of a ping.  Compressed pings (`compressed_images: True`, a sensor_msgs/CompressedImage
        whose `.data` holds the PNG/JPEG bytes) are decoded on the host exactly like the reference does
        (feature_extraction.py:210-213: cv2.imdecode as BGR, then BGR -> gray) -- or, with `decode_on_device`, on the GPU
        when sonar_slam_b200.jpeg or .png accepts the stream (the same image); anything else is taken as the decoded
        [num_ranges, num_beams] array (the reference's ros_numpy.image_to_numpy branch, :217)."""
        img = getattr(sonar_msg, "image", None)
        if img is None:
            img = sonar_msg.ping
        data = getattr(img, "data", None)
        if self.compressed_images and isinstance(data, (bytes, bytearray, memoryview)):
            if self.decode_on_device:
                from .. import jpeg, png
                codec = png if bytes(data[:8]) == png.SIGNATURE else jpeg
                info = codec.inspect([data])[0]
                if info[0] == codec.OK:
                    out, st = codec.decode_host([data], info[1], info[2])
                    if st[0] == codec.OK:
                        return out[0]
                # rejected, or data the device calls corrupt (e.g. truncated: libjpeg-turbo pads it and warns):
                # the reference's own decoder decides, as it does without decode_on_device
            import cv2  # the reference's own decoder; only needed for compressed bags
            buf = np.frombuffer(data, np.uint8)
            dec = cv2.imdecode(buf, cv2.IMREAD_COLOR)
            if dec is None:
                raise ValueError("FeatureExtraction: the compressed ping could not be decoded")
            img = cv2.cvtColor(np.array(dec).astype(np.uint8), cv2.COLOR_BGR2GRAY)
        return np.ascontiguousarray(img)

    def callback(self, sonar_msg):
        if sonar_msg.ping_id % self.skip != 0:
            self.feature_img = None
            nan = np.array([[np.nan, np.nan]])
            return self.publish_features(sonar_msg, nan)

        img = self.ping_image(sonar_msg)
        if img.dtype != np.uint8 or img.ndim != 2:
            raise TypeError("FeatureExtraction.callback: the ping image must be uint8 [num_ranges, num_beams]")
        self.generate_map_xy(sonar_msg)

        # CFAR + amplitude gate (feature_extraction.py:223-224), on the device
        if self.detector is None:
            self.configure()
        prm = self.detector.params[self.alg]
        train_hs, guard_hs, tau = prm[0], prm[1], prm[-1]
        rank = prm[2] if self.alg == "OS" else 0
        ctx = _lib.default_context()
        R, B = img.shape
        mask = np.empty((R, B), np.uint8)
        _lib.check(ctx.lib.sfe_cfar_host(ctx.handle, _lib.ptr(img), 0, 1, R, B, _ALG[self.alg], int(train_hs),
                                         int(guard_hs), int(rank), float(tau), 1, float(self.threshold),
                                         _lib.ptr(mask), None), "FeatureExtraction: cfar")
        maps = self.device_maps(ctx, B)
        if self.render_feature_img:  # cv2.remap(img) + applyColorMap(JET), published as bgr8 (:226-228)
            from .. import feature_image
            from . import conversions
            self.feature_img = feature_image.render_host(maps, img, ctx=ctx)[0]
            self.feature_img_msg = conversions.numpy_to_image(self.feature_img, "bgr8")
        # remap + nonzero + metres (:231-238)
        cap = self.rows * self.cols
        ij = np.empty((cap, 2), np.int32)
        xy = np.empty((cap, 2), np.float32)
        cnt = np.zeros(1, np.int32)
        _lib.check(ctx.lib.sfe_cart_points_host(ctx.handle, maps.handle, _lib.ptr(mask), 1, cap, _lib.ptr(ij),
                                                _lib.ptr(xy), _lib.ptr(cnt)), "FeatureExtraction: cart_points")
        k = int(cnt[0])
        self.locs = ij[:k].astype(np.int64)
        points = xy[:k].copy()

        # filters (:241-249)
        if len(points) and self.resolution > 0:
            points = pcl.downsample(points, self.resolution)
        if self.outlier_filter_min_points > 1 and len(points) > 0:
            points = pcl.remove_outlier(points, self.outlier_filter_radius, self.outlier_filter_min_points)
        return self.publish_features(sonar_msg, points)

    def callback_batch(self, sonar_msgs, max_frames=256):
        """callback() over a sequence of pings: returns the list of `feature_msg`s that calling callback on each
        message in turn would leave, byte for byte, and leaves `points` / `feature_msg` as the last call would
        (`locs` and the feature images are not produced).  The pings that are not skipped go through the batched front
        end (pipeline.FrontEnd) with its scan match off, at most `max_frames` per call: streams that sonar_slam_b200.jpeg
        or .png accepts as run_jpeg_host / run_png_host, everything else decoded by ping_image and sent through
        run_host; each geometry is a front-end geometry (add_geometry).  A ping whose Cartesian cloud overflows the
        front end's cap_points, or whose stream the device decoder rejects after all, takes callback()."""
        from .. import jpeg, png
        msgs = list(sonar_msgs)
        points = [None] * len(msgs)
        if self.detector is None:
            self.configure()
        ctx = _lib.default_context()
        # the pings with device work, by how they reach the device: (message index, geometry maps, image or stream)
        groups = {jpeg: [], png: [], None: []}
        for i, m in enumerate(msgs):
            if m.ping_id % self.skip != 0:
                points[i] = np.array([[np.nan, np.nan]])
                continue
            img = getattr(m, "image", None)
            data = getattr(m.ping if img is None else img, "data", None)
            codec = None
            if self.compressed_images and isinstance(data, (bytes, bytearray, memoryview)):
                codec = png if bytes(data[:8]) == png.SIGNATURE else jpeg
                info = codec.inspect([data])[0]
                if info[0] == codec.OK:
                    R, B, img = int(info[1]), int(info[2]), bytes(data)
                else:
                    codec = None
            if codec is None:
                img = self.ping_image(m)
                if img.dtype != np.uint8 or img.ndim != 2:
                    raise TypeError("FeatureExtraction.callback: the ping image must be uint8 [num_ranges, num_beams]")
                R, B = img.shape
            self.generate_map_xy(m)
            groups[codec].append((i, self._batch_maps(ctx, B), img))
        for codec, items in groups.items():
            for s in range(0, len(items), max_frames):
                part = items[s:s + max_frames]
                try:
                    clouds = self._batch_clouds(ctx, codec, part, max_frames)
                except _lib.SonarFEError:
                    if codec is None:
                        raise
                    clouds = [None] * len(part)  # a stream the device decoder rejects: callback's own path decides
                for (i, _, _), c in zip(part, clouds):
                    points[i] = c if c is not None else self.callback(msgs[i])
        out = []
        for m, p in zip(msgs, points):
            self.publish_features(m, p)
            out.append(self.feature_msg)
        return out

    def _batch_maps(self, ctx, num_beams):
        """The device maps of the geometry generate_map_xy set last, kept for later batches."""
        cache = self.__dict__.setdefault("_batch_maps_cache", {})
        key = (id(ctx), self.rows, self.cols, num_beams, self.width, self.height, self.res)
        if key not in cache:
            cache[key] = _lib.Maps(ctx, self.map_x, self.map_y, self.rows, num_beams, self.width, self.height)
        return cache[key]

    def _batch_clouds(self, ctx, codec, part, max_frames):
        """The filtered clouds of `part` ((index, maps, image or stream) each) from one front-end call per group of
        geometries that share frame slots; None where a Cartesian cloud overflowed cap_points."""
        from .. import pipeline
        prm = self.detector.params[self.alg]
        kw = dict(cfar_alg=_ALG[self.alg], train_hs=int(prm[0]), guard_hs=int(prm[1]),
                  rank=int(prm[2]) if self.alg == "OS" else 0, tau=float(prm[-1]), gate_enable=1,
                  gate_threshold=float(self.threshold), resolution=float(self.resolution),
                  outlier_radius=float(self.outlier_filter_radius),
                  outlier_min_points=int(self.outlier_filter_min_points), flip_lateral=0)
        # a front end's geometry 0 sets its frame slots; every other geometry must fit them
        heads = []
        for maps in sorted({id(m): m for _, m, _ in part}.values(), key=lambda m: -m.R * m.B):
            home = next((h for h in heads if maps.R <= h[0].R and maps.B <= h[0].B), None)
            if home is None:
                heads.append([maps])
            else:
                home.append(maps)
        cache = self.__dict__.setdefault("_batch_frontends", {})
        clouds = [None] * len(part)
        for geos in heads:
            key = (tuple(id(m) for m in geos), max_frames, tuple(sorted(kw.items())))
            if key not in cache:
                fe = pipeline.FrontEnd(ctx, geos[0], max_frames, **kw)
                for m in geos[1:]:
                    fe.add_geometry(m)
                fe.set_scan_match(False)
                cache[key] = fe
            fe = cache[key]
            gid = {id(m): g for g, m in enumerate(geos)}
            sel = [k for k, (_, m, _) in enumerate(part) if id(m) in gid]
            geometry = np.array([gid[id(part[k][1])] for k in sel], np.int32)
            frames = [part[k][2] for k in sel]
            poses = np.zeros((len(sel), 3))
            if codec is not None:
                run = fe.run_jpeg_host if codec.__name__.endswith("jpeg") else fe.run_png_host
                res = run(frames, poses, geometry=geometry, clouds=True)
            else:
                res = fe.run_host(frames, poses, geometry=geometry, clouds=True)
            off = res["cloud_offsets"]
            for j, k in enumerate(sel):
                if res["status"][j] != _lib.ICP_TOO_LARGE:
                    clouds[k] = res["clouds"][off[j]:off[j + 1]].copy()
        return clouds
