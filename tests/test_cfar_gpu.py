"""GPU parity: libsonarfe CFAR (through the C ABI) vs the CPU oracle -- bit-exact masks and
bit-exact float32 threshold images, for every variant, both dtypes, streaming and general path."""
import hashlib

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from sonar_slam_b200 import ops, synth

pytestmark = pytest.mark.gpu

TAU = {"CA": 2.3701490070915554, "SOCA": 2.749063720096473, "GOCA": 2.121926842646487, "OS": 9.137608674642355}
ALGS = ["CA", "SOCA", "GOCA", "OS"]


def _oracle_batch(alg, imgs, T, G, k, tau, gate=None, want_thr=False):
    masks, thrs = [], []
    for im in imgs:
        m, t = orc.cfar(alg, im, T, G, k, tau, want_thr=want_thr)
        m = np.ascontiguousarray(m)
        if gate is not None:
            m = m & (im > gate)
        masks.append(m)
        thrs.append(np.ascontiguousarray(t) if want_thr else None)
    return np.stack(masks), (np.stack(thrs) if want_thr else None)


def _unpack_bits(bits, B):
    w = bits.cpu().numpy().view(np.uint32)
    out = ((w[..., :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(np.uint8)
    return out.reshape(w.shape[0], w.shape[1], -1)[..., :B]


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_default_config_batch(gpu_ctx, alg, dtype):
    imgs = synth.make_frames(range(10, 16))                    # 6 x 512 x 512 uint8
    dev = torch.from_numpy(imgs).cuda().to(dtype)
    out = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10, want_thr=True, want_bits=True)
    want_m, want_t = _oracle_batch(alg, imgs, 20, 5, 10, TAU[alg], want_thr=True)
    assert np.array_equal(out["mask"].cpu().numpy(), want_m)
    assert np.array_equal(out["thr"].cpu().numpy().view(np.uint32), want_t.view(np.uint32))
    assert np.array_equal(_unpack_bits(out["bits"], 512), want_m)
    # plain variant (no threshold image) goes through the float32-estimate + exact-fallback compare
    out2 = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10)
    assert np.array_equal(out2["mask"].cpu().numpy(), want_m)


@pytest.mark.parametrize("alg", ALGS)
def test_gate_fused(gpu_ctx, alg):
    imgs = synth.make_frames([1, 2])
    for dtype in (torch.uint8, torch.float32):
        dev = torch.from_numpy(imgs).cuda().to(dtype)
        got = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10, gate=65, want_bits=True)
        want, _ = _oracle_batch(alg, imgs, 20, 5, 10, TAU[alg], gate=65)
        assert np.array_equal(got["mask"].cpu().numpy(), want)
        assert np.array_equal(_unpack_bits(got["bits"], 512), want)


@pytest.mark.parametrize("alg", ALGS)
def test_golden_masks_from_reference(gpu_ctx, alg, golden_dir):
    g = np.load(f"{golden_dir}/cfar_masks.npz")
    img = torch.from_numpy(synth.make_frame(1)).cuda()
    out = ops.cfar(img, alg, 20, 5, TAU[alg], k=10, want_thr=True)
    m = out["mask"][0].cpu().numpy()
    assert np.array_equal(np.packbits(m), g[alg])
    thr = out["thr"][0].cpu().numpy()
    assert hashlib.sha256(thr.tobytes()).hexdigest() == str(g[alg + "_thr_sha256"])


@pytest.mark.parametrize("alg", ALGS)
def test_non_integer_float_images_are_bit_exact(gpu_ctx, alg):
    """Fractional / huge / negative cells: the streaming kernel must hand those strips to the
    sequential-order kernel; results stay bit-identical to the reference arithmetic."""
    rng = np.random.default_rng(5)
    imgs = (rng.rayleigh(18.0, (3, 512, 512)) + rng.random((3, 512, 512))).astype(np.float32)
    imgs[1, :, :128] = np.rint(imgs[1, :, :128])               # one clean strip inside a dirty frame
    imgs[2] = np.rint(imgs[2])
    imgs[2, 300, 200] = 1.0e6                                   # integer but beyond the exact-sum range
    imgs[2, 17, 5] = -3.0
    dev = torch.from_numpy(imgs).cuda()
    out = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10, want_thr=True)
    want_m, want_t = _oracle_batch(alg, imgs, 20, 5, 10, TAU[alg], want_thr=True)
    assert np.array_equal(out["mask"].cpu().numpy(), want_m)
    assert np.array_equal(out["thr"].cpu().numpy().view(np.uint32), want_t.view(np.uint32))
    out = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10)
    assert np.array_equal(out["mask"].cpu().numpy(), want_m)


@pytest.mark.parametrize("shape,T,G,k", [((1, 512, 512), 12, 3, 5), ((2, 100, 77), 20, 5, 39), ((1, 51, 16), 20, 5, 0),
                                          ((1, 50, 16), 20, 5, 0), ((3, 131, 130), 4, 0, 7), ((1, 640, 256), 20, 5, 10),
                                          ((2, 200, 48), 20, 5, 3)])
def test_general_shapes_and_windows(gpu_ctx, shape, T, G, k):
    rng = np.random.default_rng(11)
    imgs = rng.integers(0, 256, shape).astype(np.uint8)
    for alg in ALGS:
        for dtype in (torch.uint8, torch.float32):
            dev = torch.from_numpy(imgs).cuda().to(dtype)
            out = ops.cfar(dev, alg, T, G, 1.7, k=k, want_thr=True, want_bits=True)
            want_m, want_t = _oracle_batch(alg, imgs, T, G, k, 1.7, want_thr=True)
            assert np.array_equal(out["mask"].cpu().numpy(), want_m), (alg, dtype, shape)
            assert np.array_equal(out["thr"].cpu().numpy().view(np.uint32), want_t.view(np.uint32))
            assert np.array_equal(_unpack_bits(out["bits"], shape[2]), want_m)


def test_threshold_on_the_knife_edge(gpu_ctx):
    """Cells exactly at / one ulp around tau*S/T: the float32 pre-test must defer to double."""
    R, B = 512, 128
    img = np.full((R, B), 40, np.float32)
    tau = 1.25                                                  # threshold = 1.25*800/20 = 50 exactly
    img[100:110, :] = 50                                        # equal -> not detected (strict >)
    img[200:203, :] = 51
    dev = torch.from_numpy(img).cuda()
    for alg in ("CA", "SOCA", "GOCA"):
        got = ops.cfar(dev, alg, 20, 5, tau)["mask"][0].cpu().numpy()
        want = np.ascontiguousarray(orc.cfar(alg, img, 20, 5, 0, tau)[0])
        assert np.array_equal(got, want), alg
    for tau in (np.nextafter(1.25, 2.0), np.nextafter(1.25, 0.0), 1.2500001, 1.2499999):
        got = ops.cfar(dev, "SOCA", 20, 5, float(tau))["mask"][0].cpu().numpy()
        want = np.ascontiguousarray(orc.cfar("SOCA", img, 20, 5, 0, float(tau))[0])
        assert np.array_equal(got, want), tau


def test_empty_and_degenerate(gpu_ctx):
    z = torch.zeros((0, 512, 512), dtype=torch.uint8, device="cuda")
    assert ops.cfar(z, "SOCA", 20, 5, 2.0)["mask"].shape == (0, 512, 512)
    flat = torch.zeros((1, 512, 512), dtype=torch.uint8, device="cuda")
    assert int(ops.cfar(flat, "SOCA", 20, 5, 2.0)["mask"].sum()) == 0       # 0 > tau*0 is false
    with pytest.raises(Exception):
        ops.cfar(flat, "OS", 20, 5, 2.0, k=40)                              # rank outside [0, 2T)


def test_drop_in_module_and_class(gpu_ctx):
    """bruce_slam.cfar / CFAR as the node uses them (feature_extraction.py:223-224)."""
    from sonar_slam_b200.bruce_slam.CFAR import CFAR
    from sonar_slam_b200.bruce_slam import cfar
    img = synth.make_frame(1)
    det = CFAR(40, 10, 0.1, 10)
    for alg in ALGS:
        peaks = det.detect(img, alg)
        assert peaks.dtype == np.uint8 and peaks.shape == img.shape and peaks.flags["F_CONTIGUOUS"]
        want, want_t = orc.cfar(alg, img, 20, 5, 10, TAU[alg], want_thr=True)
        assert np.array_equal(peaks, want)
        peaks &= img > 65                                       # the node's in-place gate must work on our array
        m2, t2 = det.detect2(img.astype(np.float64), alg)       # any real dtype, like pybind
        assert np.array_equal(m2, want) and np.array_equal(t2, want_t)
    assert np.array_equal(cfar.soca(img, 20, 5, 2.0), orc.cfar("SOCA", img, 20, 5, 0, 2.0)[0])


def test_large_batch_checksum_properties(gpu_ctx):
    """Config-2 scale (here 256 frames): size-independent checks instead of a CPU oracle pass:
    per-frame results are independent of batch position and of the dtype the frame is stored in."""
    g = torch.Generator(device="cuda").manual_seed(3)
    u = torch.rand((256, 512, 512), device="cuda", generator=g).clamp_min(1e-7)
    imgs = torch.clamp(torch.round(18.0 * torch.sqrt(-2.0 * torch.log(u))), 0, 255).to(torch.uint8)
    a = ops.cfar(imgs, "SOCA", 20, 5, TAU["SOCA"], gate=65)["mask"]
    b = ops.cfar(imgs.float(), "SOCA", 20, 5, TAU["SOCA"], gate=65)["mask"]
    assert torch.equal(a, b)
    perm = torch.randperm(256, device="cuda", generator=g)
    c = ops.cfar(imgs[perm].contiguous(), "SOCA", 20, 5, TAU["SOCA"], gate=65)["mask"]
    assert torch.equal(c, a[perm])
    assert int(a[:, :25].sum()) == 0 and int(a[:, -25:].sum()) == 0
    idx = [0, 100, 255]
    want, _ = _oracle_batch("SOCA", imgs[idx].cpu().numpy(), 20, 5, 0, TAU["SOCA"], gate=65)
    assert np.array_equal(a[idx].cpu().numpy(), want)


def _pack_bits(masks):
    """0/1 masks [F, R, B] as the bit plane sfe_cfar_dev writes: [F, R, ceil(B/32)] words, bit b & 31 of word b >> 5
    is beam b, the bits past B are 0."""
    F, R, B = masks.shape
    padded = np.zeros((F, R, (B + 31) // 32 * 32), np.uint8)
    padded[..., :B] = masks
    return np.packbits(padded, axis=-1, bitorder="little").view("<u4")


@pytest.mark.parametrize("shape", [(3, 512, 512), (2, 512, 528), (2, 100, 256), (1, 77, 1024), (2, 333, 48),
                                   (1, 51, 16), (2, 512, 1040)])
@pytest.mark.parametrize("gate", [None, 14, 15, 16, 65, 127, 128])
def test_u8_gated_four_beam_kernel(gpu_ctx, shape, gate):
    """The uint8 streaming kernels against the oracle, each reached through cfar_run's own choice: the gated
    4-beams-per-thread kernel (cfar_u8_gate4_kernel, detections decided in a rare branch) when the pass table's
    least entry g_min lies in [16, 128], else the table kernel.  A zero window sum has entry 1 for any finite tau, so
    g_min = max(1, floor(gate) + 1): gates 15 .. 127 take the gate kernel; no gate, 14 and 128 the table kernel.
    Speckle frames (few candidates), bright frames (every row takes the branch), strips that end inside a 512-beam
    block, images shorter than the window; masks and bit planes, alone and together."""
    g_min = 1 if gate is None else max(1, int(np.floor(gate)) + 1)
    kernel = "gate4" if 16 <= g_min <= 128 else "table"
    rng = np.random.default_rng(shape[1] * 7 + shape[2] + (gate or 0))
    speckle = np.clip(np.rint(rng.rayleigh(18.0, shape)), 0, 255).astype(np.uint8)
    bright = rng.integers(0, 256, shape).astype(np.uint8)
    for imgs in (speckle, bright):
        dev = torch.from_numpy(imgs).cuda()
        for alg in ("CA", "SOCA", "GOCA"):
            a = ops.cfar(dev, alg, 20, 5, TAU[alg], gate=gate, want_mask=True, want_bits=True)
            b = ops.cfar(dev, alg, 20, 5, TAU[alg], gate=gate, want_mask=False, want_bits=True)
            c = ops.cfar(dev, alg, 20, 5, TAU[alg], gate=gate, want_mask=True)
            want, _ = _oracle_batch(alg, imgs, 20, 5, 0, TAU[alg], gate=gate)
            tag = (kernel, alg, shape, gate)
            assert np.array_equal(a["mask"].cpu().numpy(), want), tag
            assert np.array_equal(c["mask"].cpu().numpy(), want), tag
            assert np.array_equal(a["bits"].cpu().numpy().view(np.uint32), _pack_bits(want)), tag
            assert np.array_equal(b["bits"].cpu().numpy().view(np.uint32), _pack_bits(want)), tag


def test_float_images_with_nan_and_inf(gpu_ctx):
    """A NaN / +-inf cell must hand its strip to the sequential-order kernel: like cfar.cpp, rows whose windows
    contain the cell detect nothing (comparisons with NaN are false), rows after it detect again."""
    rng = np.random.default_rng(9)
    imgs = np.rint(rng.rayleigh(18.0, (3, 512, 256))).astype(np.float32)
    imgs[0, 100, 7] = np.nan
    imgs[0, 300, 200] = np.inf
    imgs[1, 250, 130] = -np.inf
    imgs[2, 40:44, 3] = np.nan
    imgs[:, 400:403, :] += 150.0                                # detections below every special cell
    dev = torch.from_numpy(imgs).cuda()
    for alg in ("CA", "SOCA", "GOCA"):   # (std::nth_element over NaN is undefined behaviour in the reference's OS)
        want_m, want_t = _oracle_batch(alg, imgs, 20, 5, 10, TAU[alg], want_thr=True)
        out = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10)
        assert np.array_equal(out["mask"].cpu().numpy(), want_m), alg
        out = ops.cfar(dev, alg, 20, 5, TAU[alg], k=10, want_thr=True)
        assert np.array_equal(out["mask"].cpu().numpy(), want_m), alg
        thr = out["thr"].cpu().numpy()
        nan = np.isnan(want_t)                                  # NaN thresholds: same places (payload bits are the FPU's)
        assert np.array_equal(np.isnan(thr), nan), alg
        assert np.array_equal(thr[~nan].view(np.uint32), want_t[~nan].view(np.uint32)), alg
    assert want_m[0, 400:403, 7].any()                          # the beam recovers once the NaN left the window


def test_lut_cache_is_per_context(gpu_ctx):
    """Two contexts on one thread, different parameters, interleaved calls: each keeps its own table."""
    from sonar_slam_b200 import _lib
    imgs = synth.make_frames([4, 5])
    dev = torch.from_numpy(imgs).cuda()
    s2 = torch.cuda.Stream()
    other = _lib.Context(0, s2.cuda_stream)
    w65, _ = _oracle_batch("SOCA", imgs, 20, 5, 0, TAU["SOCA"], gate=65)
    w90, _ = _oracle_batch("SOCA", imgs, 20, 5, 0, 3.5, gate=90)
    for _ in range(3):
        a = ops.cfar(dev, "SOCA", 20, 5, TAU["SOCA"], gate=65)
        with torch.cuda.stream(s2):
            b = ops.cfar(dev, "SOCA", 20, 5, 3.5, gate=90, ctx=other)
        torch.cuda.synchronize()
        assert np.array_equal(a["mask"].cpu().numpy(), w65) and np.array_equal(b["mask"].cpu().numpy(), w90)
