"""The mask branch on the distinct live boxes only: the row plan (upsnet_mask_rows) against a torch restatement, the
count-bounded launches of the TMA-fed conv (upsnet_igemm_forward with n_dev) and of the pair ROIAlign
(upsnet_roi_align_fpn_forward with n_dev) against their unbounded launches, and the static engine with the plan on vs off.
Every bounded result below the count must be bit-identical to the unbounded one: a skipped tile changes no arithmetic.
Own file = own process (a trap in a tensor-core kernel poisons the CUDA context)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
NS = (0, 1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256)   # around tile edges of 1..64 rows


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


@pytest.fixture()
def pair_mode():
    import upsnet_b200 as U
    U.set_precision("bf16x3")
    yield U
    U.set_precision("fp32")


def _count(n, dev):
    return torch.tensor(n, dtype=torch.int32, device=dev)


# ---------------------------------------------------------------------------------------------------------------------
# row plan
# ---------------------------------------------------------------------------------------------------------------------
def _plan_ref(b1, n1, b2, n2):
    cap1, cap2 = b1.shape[0], b2.shape[0]
    rows = torch.zeros((cap1 + cap2, 5), dtype=torch.float32)
    rows[:n1] = b1[:n1]
    d = b1[:n1].contiguous().view(torch.int32)
    pan = torch.zeros(cap2, dtype=torch.int32)
    u = n1
    for j in range(n2):
        hit = (d == b2[j].contiguous().view(torch.int32)).all(1).nonzero()
        if hit.numel():
            pan[j] = int(hit[0, 0])
        else:
            rows[u] = b2[j]
            pan[j] = u
            u += 1
    return rows, u, pan


def _boxes(rng, n):
    xy = rng.uniform(0, 1500, (n, 2))
    wh = rng.uniform(4, 300, (n, 2))
    return torch.from_numpy(np.concatenate([np.zeros((n, 1)), xy, xy + wh], 1).astype(np.float32))


def _plan_cases():
    rng = np.random.default_rng(3)
    cap = 128
    out = []
    b1, b2 = _boxes(rng, cap), _boxes(rng, cap)
    out.append(("no_overlap", b1, 100, b2, 90))
    b2f = b1[torch.from_numpy(rng.permutation(cap))].clone()
    out.append(("full_overlap", b1, 128, b2f, 100))
    out.append(("n1_zero", b1, 0, b2, 60))
    out.append(("n2_zero", b1, 70, b2, 0))
    mix = b2.clone()
    mix[::2] = b1[torch.from_numpy(rng.choice(cap, cap // 2, replace=False))]
    out.append(("both_full", b1, 128, mix, 128))
    dup = b2.clone()
    dup[5] = dup[3]; dup[6] = dup[3]; dup[9] = b1[7]; dup[10] = b1[7]
    out.append(("duplicates_in_b2", b1, 50, dup, 40))
    ulp = b1[:40].clone()
    ulp = torch.cat([ulp, torch.zeros((cap - 40, 5))])
    ulp[4, 3] = float(np.nextafter(np.float32(ulp[4, 3]), np.float32(np.inf)))
    ulp[11, 1] = float(np.nextafter(np.float32(ulp[11, 1]), np.float32(-np.inf)))
    out.append(("one_ulp", b1, 60, ulp, 40))
    return out


@pytest.mark.parametrize("case", _plan_cases(), ids=lambda c: c[0])
def test_row_plan_vs_torch(dev, case):
    from upsnet_b200 import operators as ops
    _, b1, n1, b2, n2 = case
    want_rows, want_u, want_pan = _plan_ref(b1, n1, b2, n2)
    rows, u, pan = ops.mask_rows(b1.to(dev), _count(n1, dev), b2.to(dev), _count(n2, dev))
    rows, u, pan = rows.cpu(), int(u), pan.cpu()
    assert u == want_u
    assert torch.equal(rows[:u].view(torch.int32), want_rows[:u].view(torch.int32))
    assert torch.equal(rows[u:], torch.zeros_like(rows[u:]))
    assert torch.equal(pan[:n2], want_pan[:n2])
    assert (pan[n2:] == 0).all()
    if case[0] == "one_ulp":
        assert pan[4] >= n1 and pan[11] >= n1 and pan[5] == 5     # one ulp apart: not merged


# ---------------------------------------------------------------------------------------------------------------------
# count-bounded TMA conv and pair ROIAlign: bounded vs unbounded launch into sentinel-filled outputs
# ---------------------------------------------------------------------------------------------------------------------
def _conv_raw(x_store, w, b, y, N, H, W, Cin, Cout, k, pad, pair_out, flags, n_dev):
    from upsnet_b200 import _lib, operators as ops
    from upsnet_b200._lib import check, lib, ptr, stream_ptr
    packed = ops._packed_weight(w)
    check(lib().upsnet_igemm_forward(ptr(x_store), ptr(None), ptr(None), ptr(packed), ptr(b), ptr(None), ptr(y),
                                     N, H, W, Cin, Cout, k, k, 1, 1, pad, pad, 1, 1, _lib.LAYOUT_NHWC, _lib.DTYPE_PAIR,
                                     _lib.DTYPE_PAIR if pair_out else _lib.DTYPE_F32, flags, _lib.PREC_BF16X3,
                                     ptr(n_dev), stream_ptr(x_store.device)), "igemm_forward")


def _sentinel_like(shape, dtype, dev):
    return torch.full(shape, -12345.0, dtype=dtype, device=dev)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _check_bounded(full, bounded, n, sentinel, exact):
    """Rows < n bit-identical to the full launch; from the first skipped tile on, rows untouched; rows of the tile that
    straddles n computed in full (a tile holds at most 128 pixels, so it spans fewer than 128 rows beyond n).  exact: one
    row per block (ROIAlign), nothing beyond n is written."""
    N = full.shape[0]
    fb, bb, sb = _bits(full), _bits(bounded), _bits(sentinel)
    assert torch.equal(bb[:n], fb[:n])
    untouched = (bb == sb).flatten(1).all(1).cpu()
    r0 = n
    while r0 < N and not bool(untouched[r0]):
        r0 += 1
    assert bool(untouched[r0:].all())
    assert torch.equal(bb[n:r0], fb[n:r0])
    assert r0 - n < 128 and (r0 < N or n + 128 > N)     # whole tiles beyond n are skipped
    if exact:
        assert r0 == n


# (N, H, W, Cin, Cout, k, pair_group, pair_out): the mask head at 256 rois (its tiles hold 16 to 64 rois each) and a
# 4x4 map with 8 images per tile
CONV_SHAPES = {
    "mask_conv3x3": (256, 14, 14, 256, 256, 3, 0, True),
    "mask_deconv_pair_group": (256, 14, 14, 256, 1024, 1, 256, True),
    "mask_score_direct": (256, 14, 56, 256, 9, 1, 0, False),
    "multi_image_tiles": (256, 4, 4, 64, 128, 3, 0, True),
}


@pytest.mark.parametrize("name", list(CONV_SHAPES))
def test_bounded_conv_vs_full(dev, pair_mode, name):
    from upsnet_b200 import operators as ops
    N, H, W, Cin, Cout, k, pg, pair_out = CONV_SHAPES[name]
    g = torch.Generator(device="cpu").manual_seed(11)
    x = ops.Pair.from_float(torch.randn(N, Cin, H, W, generator=g).to(dev))
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(dev)
    b = torch.randn(Cout, generator=g).to(dev)
    pad = k // 2
    flags = 1 | (((pg // 64) & 0xfff) << 8)
    shape = (N, H, W, 2 * Cout) if pair_out else (N, H, W, Cout)
    dt = torch.bfloat16 if pair_out else torch.float32
    full = _sentinel_like(shape, dt, dev)
    _conv_raw(x.store, w, b, full, N, H, W, Cin, Cout, k, pad, pair_out, flags, None)
    for n in NS:
        sent = _sentinel_like(shape, dt, dev)
        out = sent.clone()
        _conv_raw(x.store, w, b, out, N, H, W, Cin, Cout, k, pad, pair_out, flags, _count(n, dev))
        torch.cuda.synchronize()
        _check_bounded(full, out, n, sent, False)


def test_bounded_pair_roi_align(dev, pair_mode):
    from upsnet_b200 import _lib, operators as ops
    from upsnet_b200._lib import check, lib, ptr, stream_ptr
    g = torch.Generator(device="cpu").manual_seed(12)
    Cc, R, P = 256, 256, 14
    feats = [ops.Pair.from_float(torch.randn(1, Cc, 64 >> l, 128 >> l, generator=g).to(dev)) for l in range(4)]
    rois = _boxes(np.random.default_rng(4), R)
    rois[:, 1:] = rois[:, 1:] / 1800 * torch.tensor([511, 255, 511, 255])
    rois = rois.to(dev)
    fp = (C.c_void_p * 4)(*[f.store.data_ptr() for f in feats])
    hs = (C.c_int * 4)(*[f.shape[2] for f in feats]); ws = (C.c_int * 4)(*[f.shape[3] for f in feats])
    sc = (C.c_float * 4)(*[0.25, 0.125, 0.0625, 0.03125])

    def run(out, n_dev):
        check(lib().upsnet_roi_align_fpn_forward(fp, hs, ws, sc, 1, Cc, _lib.LAYOUT_NHWC, _lib.DTYPE_PAIR, ptr(rois), R, P, P,
                                                 2, ptr(out), ptr(None), ptr(n_dev), stream_ptr(dev)), "fpn_roi_align")
    full = _sentinel_like((R, P, P, 2 * Cc), torch.bfloat16, dev)
    run(full, None)
    for n in NS:
        sent = _sentinel_like((R, P, P, 2 * Cc), torch.bfloat16, dev)
        out = sent.clone()
        run(out, _count(n, dev))
        torch.cuda.synchronize()
        _check_bounded(full, out, n, sent, True)


# ---------------------------------------------------------------------------------------------------------------------
# static engine: plan on vs off, and one captured graph replayed on images with different counts
# ---------------------------------------------------------------------------------------------------------------------
H_IMG, W_IMG = 256, 512
# (image seed, input scale).  The detection MaskROI runs at score threshold 0.5 so that its count varies with the image
# (the last image keeps ~40 detections and only the dummy panoptic candidate, whose zero box matches no detection: u > n1)
IMAGES = ((0, 1.0), (1, 1.0), (2, 0.25), (3, 0.05))


@pytest.fixture(scope="module")
def engine(dev):
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    U.set_precision("bf16x3")
    m = synthetic_model(UPSNetConfig.cityscapes_r50(), depth=(1, 1, 1, 1), seed=0, device=dev)
    m.prepare()
    m.mask_roi_static.score_thresh = 0.5
    imgs = []
    for seed, scale in IMAGES:
        inp = synthetic_input(H_IMG, W_IMG, seed=seed)
        imgs.append((inp["data"] * scale).to(dev))
    yield m, imgs, inp["im_info"][0]
    U.set_precision("fp32")


def _result(out):
    n1, n2, _ = (int(v) for v in out["counts"].tolist())
    d = out["pred_boxes"][:n1].contiguous().view(torch.int32)
    c = out["p_boxes"][:n2].contiguous().view(torch.int32)
    u = n1 + int((~(c[:, None] == d[None]).all(-1).any(-1)).sum()) if n1 else n2
    return {"counts": (n1, n2, u), "mask_probs": out["mask_probs"][:n1].clone(), "p_mask_score": out["p_mask_score"][:n2].clone(),
            "panoptic_outputs": out["panoptic_outputs"].clone(), "fcn_outputs": out["fcn_outputs"].clone(),
            "keep": out["keep"].clone()}


def _same(a, b):
    assert a["counts"] == b["counts"]
    for k in ("mask_probs", "p_mask_score"):
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
    for k in ("panoptic_outputs", "fcn_outputs", "keep"):
        assert torch.equal(a[k], b[k]), k


def _eager(m, x, info, dedup):
    m.use_cuda_graph, m.dedup_mask_rows = False, dedup
    try:
        out, _ = m._run_static(x, info)
        return _result(out)
    finally:
        m.use_cuda_graph, m.dedup_mask_rows = True, True


def test_engine_plan_on_vs_off(engine):
    m, imgs, info = engine
    seen_fresh = False
    for x in imgs:
        on, off = _eager(m, x, info, True), _eager(m, x, info, False)
        _same(on, off)
        seen_fresh |= on["counts"][2] > on["counts"][0]
    assert seen_fresh, "no image had a panoptic candidate outside the detections"


def test_graph_replay_counts_differ(engine):
    m, imgs, info = engine
    want = [_eager(m, x, info, True) for x in imgs]
    assert len({w["counts"] for w in want}) > 1, [w["counts"] for w in want]
    m._graphs = {}
    for x, w in zip(imgs, want):
        out, graph = m._run_static(x, info)
        assert graph is not None
        _same(_result(out), w)
    assert len(m._graphs) == 1
