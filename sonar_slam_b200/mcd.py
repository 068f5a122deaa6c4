"""MinCovDet of loop-closure ICP samples on the device (include/sonarfe.h: sfe_mincovdet_*).

SLAM.compute_icp_with_cov (slam.py:365-371) fits sklearn's MinCovDet(support_fraction=0.8) to the (x, y, theta)
results of up to 30 ICP runs.  The device solves many such fits in one launch (csrc/mcd.cu).  What stays on the host is
what the kernel must not re-derive: the random trial supports -- drawn from numpy's global generator exactly as
MinCovDet(random_state=None) draws them, so a seeded sequence of sklearn fits and one batch see the same supports --
and the constants, taken from the installed scipy / scikit-learn.
"""
import functools

import numpy as np

from . import _lib

TRIALS = 30                 # fast_mcd, n_samples <= 500: select_candidates(n_trials=30)
MAX_SAMPLES = 32            # one warp lane per sample
MIN_SAMPLES = 5             # compute_icp_with_cov returns "Too few samples ..." below this (slam.py:361-363)
SUPPORT_FRACTION = 0.8      # slam.py:366
OK, TOO_FEW, ZERO_COV, UNSUPPORTED, BAD_SUBSET = range(5)   # SFE_MCD_* status
FLOAT32 = 1                 # SFE_MCD_FLOAT32


def support_size(n):
    """h = int(support_fraction * n_samples) (fast_mcd)."""
    return int(SUPPORT_FRACTION * n)


@functools.lru_cache(maxsize=None)
def _constants():
    from scipy.stats import chi2
    from sklearn.covariance._robust_covariance import _consistency_factor
    c = np.zeros(MAX_SAMPLES + 1)
    for n in range(MIN_SAMPLES, MAX_SAMPLES + 1):
        c[n] = _consistency_factor(3, support_size(n) / n)
    c.setflags(write=False)
    return c, float(_consistency_factor(3, 0.975)), float(chi2(3).isf(0.025))


def constants():
    """(c_support [33], c_reweight, chi2_cut): c_support[n] = _consistency_factor(3, h / n) for n = 5..32 (what
    correct_covariance divides the distances by), _consistency_factor(3, 0.975) (reweight_covariance) and
    chi2(3).isf(0.025) (its outlier cut), from the installed libraries."""
    return _constants()


def draw_trial_supports(n, random_state=None):
    """The 30 random supports one MinCovDet(random_state).fit on n samples starts from: int8 [30, 32], row t =
    random_state.permutation(n)[:h] then -1 padding.  random_state None = numpy's global generator, which is what
    check_random_state(None) hands sklearn."""
    rs = np.random.mtrand._rand if random_state is None else random_state
    h = support_size(n)
    out = np.full((TRIALS, MAX_SAMPLES), -1, np.int8)
    for t in range(TRIALS):
        out[t, :h] = rs.permutation(n)[:h]
    return out


def pack(samples):
    """List of [n_i, 3] sample arrays -> (double [P, 32, 3], int32 n [P])."""
    X = np.zeros((len(samples), MAX_SAMPLES, 3))
    n = np.zeros(len(samples), np.int32)
    for i, s in enumerate(samples):
        s = np.asarray(s).reshape(-1, 3)
        if len(s) > MAX_SAMPLES:
            raise _lib.SonarFEError(f"MinCovDet on the device takes at most {MAX_SAMPLES} samples (got {len(s)})")
        X[i, :len(s)] = s
        n[i] = len(s)
    return X, n


def mincovdet_host(samples, n, subsets, float32=False, ctx=None):
    """Host-buffer batch fit (sfe_mincovdet_host).  samples double [P, 32, 3], n int32 [P], subsets int8 [P, 30, 32].
    float32: the samples are float32 values and numpy's float32 rules apply (compute_icp_with_cov's samples are).
    Returns dict(location [P, 3], covariance [P, 3, 3], raw_support / support uint32 [P] bit masks, status [P])."""
    ctx = ctx or _lib.default_context()
    X = np.ascontiguousarray(samples, np.float64).reshape(-1, MAX_SAMPLES, 3)
    n = np.ascontiguousarray(n, np.int32)
    sub = np.ascontiguousarray(subsets, np.int8).reshape(-1, TRIALS, MAX_SAMPLES)
    P = len(X)
    if len(n) != P or len(sub) != P:
        raise ValueError("samples, n and subsets must describe the same number of problems")
    c, c_rw, cut = constants()
    loc = np.empty((P, 3))
    cov = np.empty((P, 3, 3))
    raw, sup = np.empty(P, np.uint32), np.empty(P, np.uint32)
    st = np.empty(P, np.int32)
    _lib.check(ctx.lib.sfe_mincovdet_host(ctx.handle, _lib.ptr(X), _lib.ptr(n), _lib.ptr(sub), P, _lib.ptr(c), c_rw,
                                          cut, FLOAT32 if float32 else 0, _lib.ptr(loc), _lib.ptr(cov), _lib.ptr(raw),
                                          _lib.ptr(sup), _lib.ptr(st)), "sfe_mincovdet_host")
    return dict(location=loc, covariance=cov, raw_support=raw, support=sup, status=st)


def mask_rows(mask, n):
    """Bit mask -> boolean [n] (bit i = sample i)."""
    return ((int(mask) >> np.arange(n)) & 1).astype(bool)
