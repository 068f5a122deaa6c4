"""Scan-matching helpers of the reference's `SLAM` class, ROS- and gtsam-free
(bruce_slam/src/bruce_slam/slam.py: compute_icp :294-323, compute_icp_with_cov :325-387,
get_overlap :389-424, get_points :229-292, get_matching_cost_subroutine1 :461-570 and the shgo call around
it :683-701 / :943-961; Keyframe.transform_points slam_objects.py:178-198).

The pose-graph part of SLAM (ISAM2, PCM, keyframe logic) is out of this library's scope and stays
with the caller; `Pose2` below is a minimal stand-in for gtsam.Pose2 (x, y, theta, matrix,
between, compose) used when gtsam is not importable.
"""
import weakref

import numpy as np

from . import pcl
from .. import _lib

try:  # pragma: no cover - gtsam is not installed in the build image
    from gtsam import Pose2
except Exception:  # noqa: BLE001
    class Pose2(object):
        def __init__(self, x=0.0, y=0.0, theta=0.0):
            self._x, self._y, self._t = float(x), float(y), float(theta)

        def x(self):
            return self._x

        def y(self):
            return self._y

        def theta(self):
            return self._t

        def matrix(self):
            c, s = np.cos(self._t), np.sin(self._t)
            return np.array([[c, -s, self._x], [s, c, self._y], [0.0, 0.0, 1.0]])

        def translation(self):
            return np.array([self._x, self._y])

        def inverse(self):
            c, s = np.cos(self._t), np.sin(self._t)
            return Pose2(-(c * self._x + s * self._y), -(-s * self._x + c * self._y), -self._t)

        def compose(self, other):
            c, s = np.cos(self._t), np.sin(self._t)
            return Pose2(self._x + c * other._x - s * other._y, self._y + s * other._x + c * other._y,
                         self._t + other._t)

        def between(self, other):
            return self.inverse().compose(other)

        def __repr__(self):
            return "Pose2({:.6f}, {:.6f}, {:.6f})".format(self._x, self._y, self._t)


def transform_points(points, pose):
    """Keyframe.transform_points (slam_objects.py:178-198)."""
    if len(points) == 0:
        return np.empty_like(points, np.float32)
    T = pose.matrix().astype(np.float32)
    return points.dot(T[:2, :2].T) + T[:2, 2]


class SLAM(object):
    """Only the scan-matching surface of the reference's SLAM object."""

    def __init__(self):
        self.point_resolution = 0.5  # slam.yaml point_resolution
        self.point_noise = 0.5       # slam.py:73
        self.icp_odom_sigmas = np.array([0.1, 0.1, 0.01])
        self.icp = pcl.ICP()
        self.icp_ssm = pcl.ICP()
        self.keyframes = KeyframeList()  # a list; get_points serves it from the device-resident map
        # the two OculusProperty fields the loop-closure pre-filter reads (sonar.py:151,158)
        self.oculus = type("OculusProperty", (), {"max_range": 30.0, "horizontal_aperture": np.radians(130.0)})()

    # ---- slam.py:294-323
    def compute_icp(self, source_points, target_points, guess=None):
        guess = Pose2() if guess is None else guess
        source_points = np.array(source_points, np.float32)
        target_points = np.array(target_points, np.float32)
        message, T = self.icp.compute(source_points, target_points, guess.matrix())
        x, y = T[:2, 2]
        theta = np.arctan2(T[1, 0], T[0, 0])
        return message, Pose2(x, y, theta)

    # ---- slam.py:325-387 (the up-to-30 ICP runs go to the GPU as ONE batch instead of a timed loop)
    def compute_icp_with_cov(self, source_points, target_points, guesses):
        """slam.py:325-387: the guesses run as one ICP batch.  target_points may be the whole map (the loop-closure
        target of initialize_nonsequential_scan_matching): it is gridded once on the device and shared by every guess."""
        from sklearn.covariance import MinCovDet
        source_points = np.array(source_points, np.float32)
        target_points = np.array(target_points, np.float32)
        res = self.icp.compute_batch(source_points, target_points, [g.matrix() for g in guesses])
        sample_transforms = []
        for message, T in zip(res["messages"], res["T"]):
            if message == "success":
                x, y = T[:2, 2]
                sample_transforms.append((x, y, np.arctan2(T[1, 0], T[0, 0])))
        sample_transforms = np.array(sample_transforms)
        if len(sample_transforms) < 5:
            return "Too few samples for covariance computation", None, None, None
        try:
            fcov = MinCovDet(store_precision=False, support_fraction=0.8).fit(sample_transforms)
        except ValueError:
            return "Failed to calculate covariance", None, None, None
        m = Pose2(*fcov.location_)
        cov = fcov.covariance_
        R = m.matrix()[:2, :2]
        cov[:2, :] = R.T.dot(cov[:2, :])
        cov[:, :2] = cov[:, :2].dot(R)
        default_cov = np.diag(self.icp_odom_sigmas) ** 2
        if np.linalg.det(cov) < np.linalg.det(default_cov):
            cov = default_cov
        return "success", m, cov, sample_transforms

    def compute_icp_with_cov_batch(self, problems):
        """compute_icp_with_cov for many loop-closure candidates: `problems` is an iterable of (source_points,
        target_points, guesses); returns the list of (message, Pose2, cov, sample_transforms) that one
        compute_icp_with_cov call per candidate would return.  Every candidate's guesses go to the GPU in one ICP
        launch and every MinCovDet fit in one more (sonar_slam_b200/mcd.py).

        The fits' random trial supports are drawn here from numpy's global generator, 30 permutations per candidate
        that reaches the fit, in candidate order -- the draws MinCovDet(random_state=None) makes -- so under the same
        np.random seed this returns what the sequence of compute_icp_with_cov calls returns.  A batch of one is the
        device path for a single candidate."""
        from .. import mcd
        sources, targets, guesses = [], [], []
        for source_points, target_points, gs in problems:
            gs = list(gs)
            if len(gs) > mcd.MAX_SAMPLES:
                raise ValueError(f"compute_icp_with_cov_batch: at most {mcd.MAX_SAMPLES} guesses per candidate")
            sources.append(np.array(source_points, np.float32))
            targets.append(np.array(target_points, np.float32))
            guesses.append([g.matrix() for g in gs])
        if not sources:
            return []
        results = self.icp.compute_pairs(sources, targets, guesses)
        samples = []
        for res in results:   # slam.py:349-360, per candidate
            sample_transforms = []
            for message, T in zip(res["messages"], res["T"]):
                if message == "success":
                    x, y = T[:2, 2]
                    sample_transforms.append((x, y, np.arctan2(T[1, 0], T[0, 0])))
            samples.append(np.array(sample_transforms))
        out = [("Too few samples for covariance computation", None, None, None)] * len(samples)
        # MinCovDet.fit validates its input (finite values) before it draws; such a fit raises ValueError
        fit = []
        for i, s in enumerate(samples):
            if len(s) < mcd.MIN_SAMPLES:
                continue
            if not np.isfinite(s).all():
                out[i] = ("Failed to calculate covariance", None, None, None)
                continue
            fit.append(i)
        if not fit:
            return out
        subsets = np.stack([mcd.draw_trial_supports(len(samples[i])) for i in fit])
        X, n = mcd.pack([samples[i] for i in fit])
        f32 = np.array([samples[i].dtype == np.float32 for i in fit])
        loc, covs = np.empty((len(fit), 3)), np.empty((len(fit), 3, 3))
        status = np.empty(len(fit), np.int32)
        for flag in (True, False):   # one call per sample dtype (float32 for the shipped ICP)
            sel = np.flatnonzero(f32 == flag)
            if len(sel):
                r = mcd.mincovdet_host(X[sel], n[sel], subsets[sel], float32=flag)
                loc[sel], covs[sel], status[sel] = r["location"], r["covariance"], r["status"]
        # slam.py:372-385: unrotate into the local frame, keep the default covariance when it is bigger
        default_cov = np.diag(self.icp_odom_sigmas) ** 2
        ok = np.flatnonzero(status == mcd.OK)
        ms = [Pose2(*loc[k]) for k in ok]
        for m, k in zip(ms, ok):
            cov = covs[k]
            R = m.matrix()[:2, :2]
            cov[:2, :] = R.T.dot(cov[:2, :])
            cov[:, :2] = cov[:, :2].dot(R)
        small = np.linalg.det(covs[ok]) < np.linalg.det(default_cov) if len(ok) else np.zeros(0, bool)
        for m, k, s in zip(ms, ok, small):
            out[fit[k]] = ("success", m, default_cov if s else covs[k], samples[fit[k]])
        for k in np.flatnonzero(status != mcd.OK):
            if status[k] != mcd.ZERO_COV:
                raise RuntimeError(f"sfe_mincovdet: status {int(status[k])} for candidate {fit[k]}")
            out[fit[k]] = ("Failed to calculate covariance", None, None, None)
        return out

    # ---- slam.py:389-424
    def get_overlap(self, source_points, target_points, source_pose=None, target_pose=None, return_indices=False):
        if source_pose:
            source_points = transform_points(source_points, source_pose)
        if target_pose:
            target_points = transform_points(target_points, target_pose)
        indices, dists = pcl.match(target_points, source_points, 1, self.point_noise)
        if return_indices:
            return np.sum(indices != -1), indices
        return np.sum(indices != -1)

    # ---- slam.py:461-570
    def get_matching_cost_subroutine1(self, source_points, source_pose, target_points, target_pose,
                                      source_pose_cov=None):
        """Returns (subroutine, pose_samples) like the reference: `subroutine(x)` is the cost scipy.shgo minimises
        (minus the number of source points that fall on the dilated target grid under the pose x = [x, y, theta]
        composed onto source_pose) and every evaluation appends [pose, cost] to pose_samples.  Grid and source
        cloud live on the GPU; `subroutine.batch(xs)` scores K poses in one launch."""
        pose_samples = []
        source_points = np.ascontiguousarray(source_points, np.float32)
        target_points = np.ascontiguousarray(target_points, np.float32)

        # grid geometry: the reference's own expressions (slam.py:507-512, 522-523), evaluated by numpy
        xmin, ymin = np.min(target_points, axis=0) - 2 * self.point_noise
        xmax, ymax = np.max(target_points, axis=0) + 2 * self.point_noise
        resolution = self.point_noise / 10.0
        xs = np.arange(xmin, xmax, resolution)
        ys = np.arange(ymin, ymax, resolution)
        dilate_hs = int(np.ceil(self.point_noise / resolution))
        source_pose_info = np.linalg.inv(source_pose_cov)  # noqa: F841 (computed and unused upstream, slam.py:539)

        costmap = _lib.CostMap(_lib.default_context(), target_points, xmin, ymin, resolution, len(ys), len(xs),
                               dilate_hs)
        costmap.set_source(source_points)

        def sample_poses(x):
            delta = Pose2(*x)
            sample_source_pose = source_pose.compose(delta)
            sample_transform = target_pose.between(sample_source_pose)
            return sample_source_pose, sample_transform

        def as_row(transform):
            T = transform.matrix().astype(np.float32)  # Keyframe.transform_points, slam_objects.py:195
            return [T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]]

        def subroutine(x):
            sample_source_pose, sample_transform = sample_poses(x)
            cost = int(costmap.score(np.array([as_row(sample_transform)], np.float32))[0])
            pose_samples.append(np.r_[sample_source_pose.x(), sample_source_pose.y(), sample_source_pose.theta(), cost])
            return cost

        def batch(xs, log=True):
            """Costs of K poses [K, 3] in one launch (what a dense sampler uses instead of K shgo evaluations)."""
            xs = np.atleast_2d(np.asarray(xs, np.float64))
            poses = [sample_poses(x) for x in xs]
            costs = costmap.score(np.array([as_row(t) for _, t in poses], np.float32))
            if log:
                for (sp, _), c in zip(poses, costs):
                    pose_samples.append(np.r_[sp.x(), sp.y(), sp.theta(), int(c)])
            return costs

        subroutine.batch = batch
        subroutine.costmap = costmap
        return subroutine, pose_samples

    # ---- slam.py:667-701 (SSM) / :927-961 (NSSM): the shgo call, or one dense Sobol batch on the GPU
    def global_initialization(self, source_points, source_pose, target_points, target_pose, cov, pose_bounds,
                              initialization_params=(50, 1, 0.01), dense=0):
        """dense = 0: scipy.shgo exactly as the reference calls it (sobol sampling, n, iters, ftol), evaluating the
        GPU subroutine point by point.  dense = K > 0: score K Sobol poses inside pose_bounds in ONE launch and take
        the best (the cost is piecewise constant, so shgo's local SLSQP stage cannot improve on a sample)."""
        subroutine, pose_samples = self.get_matching_cost_subroutine1(source_points, source_pose, target_points,
                                                                      target_pose, cov)
        pose_bounds = np.asarray(pose_bounds, np.float64)
        if dense:
            from scipy.stats import qmc
            unit = qmc.Sobol(d=3, scramble=False).random(int(dense))
            xs = pose_bounds[:, 0] + unit * (pose_bounds[:, 1] - pose_bounds[:, 0])
            costs = subroutine.batch(xs)
            best = int(np.argmin(costs))  # first minimum, like a sequential scan of the samples
            return dict(success=True, x=xs[best], fun=float(costs[best]), pose_samples=np.array(pose_samples),
                        estimated_source_pose=source_pose.compose(Pose2(*xs[best])))
        from scipy.optimize import shgo
        result = shgo(func=subroutine, bounds=pose_bounds, n=initialization_params[0], iters=initialization_params[1],
                      sampling_method="sobol", minimizer_kwargs={"options": {"ftol": initialization_params[2]}})
        out = dict(success=bool(result.success), x=result.x, fun=float(result.fun), message=result.message,
                   pose_samples=np.array(pose_samples))
        if result.success:
            out["estimated_source_pose"] = source_pose.compose(Pose2(*result.x))
        return out

    # ---- slam.py:876-899 (inside initialize_nonsequential_scan_matching): field-of-view pre-filter of the targets
    def select_targets_in_fov(self, target_points, target_keys, source_frames):
        """Keep the target points (global frame) that at least one of `source_frames` could have seen, range and
        aperture inflated by 5 sigma of that keyframe's pose (keyframes need .pose and .cov).  The per-keyframe
        bounds are the reference's host expressions; the per-point test runs on the GPU (sfe_fov_select_host).
        Returns (target_points[sel], target_keys[sel], sel)."""
        target_points = np.ascontiguousarray(target_points, np.float32)
        inv_T, rb, bb = [], [], []
        for source_frame in source_frames:
            pose = self.keyframes[source_frame].pose
            cov = self.keyframes[source_frame].cov
            translation_std = np.sqrt(np.max(np.linalg.eigvals(cov[:2, :2])))
            rotation_std = np.sqrt(cov[2, 2])
            rb.append(translation_std * 5.0 + self.oculus.max_range)
            bb.append(rotation_std * 5.0 + self.oculus.horizontal_aperture * 0.5)
            T = pose.inverse().matrix().astype(np.float32)  # Keyframe.transform_points, slam_objects.py:195
            inv_T.append([T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]])
        sel = np.zeros(len(target_points), np.uint8)
        if len(target_points) and len(inv_T):
            ctx = _lib.default_context()
            inv_T = np.ascontiguousarray(inv_T, np.float32)
            rb, bb = np.ascontiguousarray(rb, np.float64), np.ascontiguousarray(bb, np.float64)
            _lib.check(ctx.lib.sfe_fov_select_host(ctx.handle, _lib.ptr(target_points), len(target_points),
                                                   _lib.ptr(inv_T), _lib.ptr(rb), _lib.ptr(bb), len(inv_T),
                                                   _lib.ptr(sel)), "sfe_fov_select_host")
        sel = sel.astype(bool)
        keys = None if target_keys is None else np.asarray(target_keys)[sel]
        return target_points[sel], keys, sel

    # ---- slam.py:229-292 for (points, pose) keyframe tuples
    def get_points(self, frames=None, ref_frame=None, return_keys=False):
        """self.keyframes: list of objects with .points ([N,2] float32) and .pose (Pose2).

        With the KeyframeList SLAM() starts with, and every selected .points a float32 [N, 2] array, the clouds are
        served from the device-resident map (KeyframeList) and only the poses travel; the results are the same.
        Otherwise (a list or dict the caller assigned, other dtypes) the lines below run on the host."""
        if frames is None:
            frames = range(len(self.keyframes))
        ref_pose = None
        if ref_frame is not None:
            ref_pose = ref_frame if isinstance(ref_frame, Pose2) else self.keyframes[ref_frame].pose
        if isinstance(self.keyframes, KeyframeList):
            frames = list(frames)
            kfs = [self.keyframes[key] for key in frames]  # IndexError here, before any device work
            if all(_resident_cloud(kf.points) for kf in kfs):
                return self._get_points_resident(frames, kfs, ref_pose, return_keys)
        all_points = [np.zeros((0, 3 if return_keys else 2), np.float32)]
        for key in frames:
            kf = self.keyframes[key]
            transf = ref_pose.between(kf.pose) if ref_pose is not None else kf.pose
            pts = transform_points(kf.points, transf)
            if return_keys:
                pts = np.c_[pts, key * np.ones((len(pts), 1))]
            all_points.append(pts)
        all_points = np.concatenate(all_points)
        if return_keys:
            return pcl.downsample(all_points[:, :2], all_points[:, (2,)], self.point_resolution)
        return pcl.downsample(all_points, self.point_resolution)

    def _get_points_resident(self, frames, kfs, ref_pose, return_keys):
        """get_points from the device-resident map: the transforms are the host path's float32 matrices, the keys its
        float64 `key * np.ones` values rounded to float32 as pcl.downsample's descriptors are."""
        if not any(len(kf.points) for kf in kfs):  # pcl.downsample hands empty input straight back
            pts = np.zeros((0, 2), np.float32)
            return (pts, np.zeros((0, 1), np.float32)) if return_keys else pts
        slots = self.keyframes.slots([kf.points for kf in kfs])
        tf = np.empty((len(kfs), 6), np.float32)
        for k, kf in enumerate(kfs):
            T = (ref_pose.between(kf.pose) if ref_pose is not None else kf.pose).matrix().astype(np.float32)
            tf[k] = T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]
        keys = np.asarray(frames, np.float64).astype(np.float32) if return_keys else None
        out = self.keyframes.map.assemble(slots, keys, tf, self.point_resolution, return_keys)
        if return_keys:
            return out[0], out[1].reshape(-1, 1)
        return out


def _resident_cloud(points):
    return isinstance(points, np.ndarray) and points.dtype == np.float32 and points.ndim == 2 and points.shape[1] == 2


class KeyframeList(list):
    """The list SLAM() keeps its keyframes in: a plain list whose keyframes' clouds are mirrored in a device-resident
    KeyframeMap (sonar_slam_b200/keyframe_map.py), created on first use on the thread's default context.

    The mirror is lazy: get_points uploads, in one append per call, every selected keyframe whose `.points` array has
    not been uploaded yet, and records which array object each slot came from.  A keyframe whose `.points` is replaced
    by another array gets a new slot.  An array edited in place after its upload is NOT detected (the reference never
    edits a keyframe's cloud; assign a new array instead)."""

    def __init__(self, *args):
        super().__init__(*args)
        self.map = None
        self._uploaded = {}  # id(points) -> (weak reference to the array, slot)

    def slots(self, clouds):
        """Slot of every array in `clouds`, appending those not stored yet (each array once)."""
        from .. import keyframe_map
        if self.map is None:
            self.map = keyframe_map.KeyframeMap(_lib.default_context())
        slots = np.empty(len(clouds), np.int32)
        new, where = [], {}
        for i, p in enumerate(clouds):
            e = self._uploaded.get(id(p))
            if e is not None and e[0]() is p:
                slots[i] = e[1]
                continue
            j = where.setdefault(id(p), len(new))
            if j == len(new):
                new.append(p)
            slots[i] = -1 - j
        if new:
            got = self.map.append(new)
            for p, s in zip(new, got):
                self._uploaded[id(p)] = (weakref.ref(p), int(s))
            pending = slots < 0
            slots[pending] = got[-1 - slots[pending]]
        return slots
