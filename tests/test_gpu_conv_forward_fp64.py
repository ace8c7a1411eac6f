"""Dense-conv forward of the inference engine -- the TMA kernel (csrc/igemm_tma.cu) and its stem, the gather kernel
(csrc/igemm_tc.cu) and the fp32 CUDA-core kernel (csrc/igemm_simt.cu) -- element by element against the float64
restatement tests/conv_grad_oracle.forward run on the device: the exact sum of the products each kernel issues, on the
operands it sees, then bias, residual, ReLU and sigmoid.  Each element is held to its own bound:
|kernel - fp64| <= c * (sum of |terms|) + slack + 1e-6, c = conv_grad_oracle.forward_c (accumulation and epilogue
adds), slack = the storage rounding of bf16 / pair outputs and the sigmoid's own rounding (conv_grad_oracle.store_slack,
SIGMOID_SLACK).  Pair outputs are also checked for a normalised hi / lo split.  Run with -s to see the worst err / bound
per (row, route).  Own file = own process (a trap in a tensor-core kernel poisons the CUDA context).

* LAYERS: one row per distinct dense signature (precision, entry, Cin, Cout, k, stride, pad, dil, bias, relu, residual,
  input storage, output storage, pair_group, sigmoid_from, n_dev set) that the inference forward of cityscapes_r50,
  coco_r50 and coco_r101_dcn calls through ops.conv2d / ops.linear / ops.stem_conv in the precisions fp32, bf16 and
  bf16x3, each at a ragged reduced size (odd H for stride 2) through the public call, with inputs in the storage the
  engine passes.  Each row asserts that its call has the row's signature.  test_census runs the inference forward of a
  synthetic model of each configuration (depth 2, 2, 2, 2) in all three precisions with recorders on ops.conv2d and
  ops.stem_conv, and fails, naming the signature, when the model calls one no row covers.  The deformable convolutions
  themselves are checked by tests/test_gpu_forward_fp64.py.
* Every row that the TMA kernel takes also runs at N tile 64 and 128 (upsnet_tma_set_tile_n, where Cout allows 128) and
  on the gather kernel (ops.USE_TMA off), checked the same way; test_routes asserts the kernel instance of each (row,
  route) from one profiler session per precision.
* Full-size rows in bf16x3 at the map sizes of 1024 x 2048 and 800 x 1344, where the tile choice is the benchmark's;
  the reference covers the first and last 8 output rows (the first and the ragged last tiles of every column).
* test_teeth: a 3x3 row through the C ABI with a copy of its packed weight in which one tap's 64-channel k-block is
  zeroed must fail the check.
tests/test_conv_grad_oracle_cpu.py shows that forward_c accepts an fp32 emulation of each precision's arithmetic and
rejects a tap one pixel off, a tap past an image's last row reading the next image, a dropped k-block, an N tile
with its neighbour's weight rows, a dropped lo*hi MMA, a truncating activation split, a stride-2 view on the odd
pixels, an up2 residual read one column off, channel co + 1's bias, a sigmoid one channel early and ReLU before the
residual.

Measured on an NVIDIA H100 80GB HBM3 (SXM, power limit 700 W), worst err / bound: bf16x3 TMA kernel 1.8e-6 (at
either N tile), gather kernel 3.0e-6 (both fc6, K = 12544), stem 1.6e-7, full-size rows <= 1.9e-6; bf16 5.4e-7 on
both kernels (the 512 -> 18 offset conv), the stem within its storage slack; fp32 CUDA-core kernel 4.0e-7.  The a-priori
constants are 10x to 100x above these, so conv_grad_oracle.FWD_TOL holds about 4x the measured values (1.2e-5, 4e-6,
1.6e-6).  The file takes 47 to 60 s there, about 33 s of it the census's three child processes.
"""
import inspect
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conv_grad_oracle as CG  # noqa: E402
import grad_oracle as G  # noqa: E402
from kernel_trace import launched_kernels_each  # noqa: E402

pytestmark = pytest.mark.gpu
PRECS = ["fp32", "bf16", "bf16x3"]
STREAM = {"fp32": "f32 nchw", "bf16": "bf16", "bf16x3": "pair"}
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)
    for k in sorted(WORST):
        print("conv forward worst err/bound %-58s %.3e (c %.2e)" % (k, *WORST[k]))


@pytest.fixture()
def engine():
    """Global engine switches, restored after every case."""
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import lib
    try:
        yield U
    finally:
        assert lib().upsnet_tma_set_tile_n(0) == 0
        ops.USE_TMA["on"] = True
        U.set_precision("fp32")


# ------------------------------------------------------------------------------------------------
# signatures
# ------------------------------------------------------------------------------------------------
def _storage(t, ops):
    if isinstance(t, ops.Pair):
        return "pair"
    if t.dtype == torch.bfloat16:
        return "bf16"
    return "f32 nchw" if t.is_contiguous() else "f32 nhwc"


def _pair1(v):
    v = tuple(v) if isinstance(v, (tuple, list)) else (v, v)
    assert v[0] == v[1], v
    return int(v[0])


def signature(prec, fn, args, y):
    """The dense signature of one ops.conv2d / ops.stem_conv call: (precision, entry, Cin, Cout, k, stride, pad, dil,
    bias, relu, residual, input storage, output storage, pair_group, sigmoid_from, n_dev set)."""
    from upsnet_b200 import operators as ops
    x, w = args["x"], args["weight"]
    if fn == "stem":
        return (prec, "stem", x.shape[1], w.shape[0], w.shape[2], 2, int(args["padding"]), 1, args["bias"] is not None,
                bool(args["relu"]), None, _storage(x, ops), _storage(y, ops), 0, None, False)
    res = None if args["residual"] is None else ("up2" if args["residual_up2"] else "same")
    return (prec, "conv2d", x.shape[1], w.shape[0], w.shape[2], _pair1(args["stride"]), _pair1(args["padding"]),
            _pair1(args["dilation"]), args["bias"] is not None, bool(args["relu"]), res, _storage(x, ops),
            _storage(y, ops), int(args["pair_group"]), args["sigmoid_from"], args["n_dev"] is not None)


def _record(monkeypatch):
    """Recorders on ops.conv2d and ops.stem_conv: -> the set the signatures of their calls go into."""
    from upsnet_b200 import _lib
    from upsnet_b200 import operators as ops
    names = {_lib.PREC_FP32_SIMT: "fp32", _lib.PREC_BF16: "bf16", _lib.PREC_BF16X3: "bf16x3"}
    seen = set()
    conv2d, stem = ops.conv2d, ops.stem_conv

    def rec(fn, f):
        sig = inspect.signature(f)

        def call(*a, **kw):
            b = sig.bind(*a, **kw)
            b.apply_defaults()
            y = f(*a, **kw)
            prec = b.arguments.get("precision")
            seen.add(signature(names[ops._PRECISION["conv"] if prec is None else prec], fn, b.arguments, y))
            return y
        return call

    monkeypatch.setattr(ops, "conv2d", rec("conv2d", conv2d))
    monkeypatch.setattr(ops, "stem_conv", rec("stem", stem))
    return seen


def _sig(prec, cin, cout, k=1, s=1, p=0, d=1, bias=True, relu=False, res=None, xin=None, out=None, pg=0, sf=None,
         ndev=False, fn="conv2d"):
    return (prec, fn, cin, cout, k, s, p, d, bias, relu, res, xin or STREAM[prec], out or STREAM[prec], pg, sf, ndev)


def _layers():
    """[(name, signature, size)]: size (N, H, W) of the input, or (R,) for a row of ops.linear."""
    rows = []
    for pr in PRECS:
        head = "f32 nchw"
        f32 = pr == "fp32"

        def add(name, size, *a, **kw):
            rows.append(("%s %s" % (pr, name), _sig(pr, *a, **kw), size))
        # stem
        if f32:
            add("stem", (1, 45, 70), 3, 64, 7, 2, 3, relu=True)
        else:
            add("stem", (1, 45, 70), 3, 64, 7, 2, 3, relu=True, xin="f32 nchw", fn="stem")
        # res2 (its block 0 reads the max-pool output: channels_last fp32 in the fp32 stream)
        nhwc = "f32 nhwc" if f32 else None
        add("res2.0 conv1", (1, 13, 22), 64, 64, relu=True, xin=nhwc)
        add("res2.0 downsample", (1, 13, 22), 64, 256, xin=nhwc)
        add("res2 3x3", (1, 13, 22), 64, 64, 3, 1, 1, relu=True)
        add("res2 conv3 +res", (1, 13, 22), 64, 256, relu=True, res="same")
        add("res2.1 conv1", (1, 13, 22), 256, 64, relu=True)
        # res3 - res5
        for stage, planes, (H, W) in ((3, 128, (13, 22)), (4, 256, (11, 19)), (5, 512, (9, 13))):
            cin = planes * 2
            add("res%d.0 conv1 s2" % stage, (1, 2 * H + 1, 2 * W), cin, planes, s=2, relu=True)
            add("res%d.0 downsample" % stage, (1, 2 * H + 1, 2 * W), cin, planes * 4, s=2)
            add("res%d conv3 +res" % stage, (1, H, W), planes, planes * 4, relu=True, res="same")
            add("res%d.1 conv1" % stage, (1, H, W), planes * 4, planes, relu=True)
        add("res3 3x3", (1, 13, 22), 128, 128, 3, 1, 1, relu=True)
        add("res4 3x3 / rpn 3x3", (1, 11, 19), 256, 256, 3, 1, 1, relu=True)
        add("res5 3x3", (1, 9, 13), 512, 512, 3, 1, 1, relu=True)
        # deformable layers' offset convs (backbone of coco_r101_dcn, semantic head)
        for cin in (128, 256, 512):
            add("offset conv %d" % cin, (1, 13, 21), cin, 18, 3, 1, 1, out=head)
        # FPN
        add("fpn_p5_1x1", (1, 9, 13), 2048, 256)
        for cin in (1024, 512, 256):
            add("fpn lateral %d +up2" % cin, (1, 14, 22), cin, 256, res="up2")
        add("fpn 3x3", (1, 13, 22), 256, 256, 3, 1, 1)
        if not f32:
            add("fpn_gap", (1,), 2048, 256, xin="f32 nchw", out=head)
        # RPN head A + 4A + A with the sigmoid on the last A (A = 3); the CUDA-core path runs the conv without it first
        add("rpn head", (1, 13, 21), 256, 18, out=head, sf=15)
        if f32:
            add("rpn head conv", (1, 13, 21), 256, 18, out=head)
        # RCNN
        add("fc6", (37,), 12544, 1024, relu=True)
        add("fc7", (37,), 1024, 1024, relu=True)
        add("cls+bbox 45", (37,), 1024, 45, out=head)
        add("cls+bbox 405", (37,), 1024, 405, out=head)
        # mask branch (n_dev = N - 1 of the rois are needed)
        add("mask 3x3", (3, 14, 14), 256, 256, 3, 1, 1, relu=True, ndev=True)
        add("mask deconv", (3, 14, 14), 256, 1024, relu=True, ndev=True, pg=256 if pr == "bf16x3" else 0)
        score = head if f32 else "f32 nhwc"
        ms = (3, 28, 28) if f32 else (3, 14, 56)          # the 4w view of the deconv output
        add("mask score 9", ms, 256, 9, out=score, ndev=True)
        add("mask score 81", ms, 256, 81, out=score, ndev=True)
        # semantic head: each level's 128-channel slice of the 1x1 score conv, the bias on P2's only
        for c in (19, 133):
            add("fcn score %d" % c, (1, 25, 26), 128, c, out=head)
            add("fcn score %d nobias" % c, (1, 13, 13), 128, c, bias=False, out=head)
    return rows


LAYERS = _layers()


# ------------------------------------------------------------------------------------------------
# one row: its call, its reference, its check
# ------------------------------------------------------------------------------------------------
def _pair_planes(store, C):
    """(hi, lo) float64 logical NCHW of a pair store [N, H, W, 2C]."""
    return tuple(store[..., i * C:(i + 1) * C].double().permute(0, 3, 1, 2) for i in (0, 1))


def _inputs(sig, size, seed, dev):
    """Random x, weight, bias, residual for the row -> (the call's arguments in the engine's storage, the values the
    kernel reads as float64)."""
    from upsnet_b200 import operators as ops
    prec, fn, cin, cout, k, s, p, d, bias, relu, res, xin, out, pg, sf, ndev = sig
    gen = torch.Generator().manual_seed(seed)
    N, H, W = (size[0], 1, 1) if len(size) == 1 else size
    x = torch.randn((N, cin, H, W), generator=gen) * (50.0 if fn == "stem" else 1.0)
    w = torch.randn((cout, cin, k, k), generator=gen) * (2.0 / (cin * k * k)) ** 0.5 / (50.0 if fn == "stem" else 1.0)
    b = torch.randn(cout, generator=gen) * 0.5 if bias else None
    Ho, Wo = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
    x, w, b = x.to(dev), w.to(dev), None if b is None else b.to(dev)
    if xin == "pair":
        xa = ops.Pair.from_float(x)
        xr = _pair_planes(xa.store, cin)
    elif xin == "bf16":
        xa = x.bfloat16().contiguous(memory_format=torch.channels_last)
        xr = xa.double()
    else:
        xa = x.contiguous(memory_format=torch.channels_last) if xin == "f32 nhwc" else x
        xr = xa.double()
    if len(size) == 1:                               # ops.linear takes [R, K] rows, or the Pair of [R, K, 1, 1]
        xa = xa if xin == "pair" else xa.reshape(N, cin)
    r = rr = None
    if res is not None:
        r = torch.randn((N, cout) + ((Ho // 2, Wo // 2) if res == "up2" else (Ho, Wo)), generator=gen).to(dev)
        if prec == "bf16x3":
            r = ops.Pair.from_float(r)
            rr = r.float().double()
        elif prec == "bf16":
            r = r.bfloat16().contiguous(memory_format=torch.channels_last)
            rr = r.double()
        else:
            rr = r.double()
    return (xa, w, b, r), (xr, w, b, rr), (N, Ho, Wo)


def _call(sig, size, args):
    from upsnet_b200 import operators as ops
    prec, fn, cin, cout, k, s, p, d, bias, relu, res, xin, out, pg, sf, ndev = sig
    x, w, b, r = args
    if fn == "stem":
        return ops.stem_conv(x, w, b, p, relu=relu, pair=out == "pair")
    if len(size) == 1:
        y = ops.linear(x, w.reshape(cout, cin), b, relu=relu, out_dtype=torch.float32 if out.startswith("f32") else None)
        return y if isinstance(y, ops.Pair) else y.reshape(y.shape[0], cout, 1, 1)
    kw = dict(stride=s, padding=p, dilation=d, residual=r, residual_up2=res == "up2", relu=relu, pair_group=pg,
              sigmoid_from=sf)
    if ndev:
        kw["n_dev"] = torch.tensor([size[0] - 1], dtype=torch.int32, device=w.device)
    if out == "f32 nchw" and prec != "fp32":
        kw["out_format"] = "nchw"
    elif out == "f32 nhwc":
        kw.update(out_format="nhwc", out_dtype=torch.float32)
    return ops.conv2d(x, w, b, **kw)


def _got(y, sig):
    """(logical float64 result laid out as the reference [N, Cout, Ho, Wo], pair store or None)."""
    from upsnet_b200 import operators as ops
    pg, cout = sig[13], sig[3]
    if not isinstance(y, ops.Pair):
        return y.double(), None
    v = y.float().double()
    if pg:      # logical [N, G, Ho, Wo * Cout / G]: column w * (Cout / G) + g holds channel g * G + c
        N, G_, Ho, W4 = v.shape
        v = v.reshape(N, G_, Ho, W4 // (cout // pg), cout // pg).permute(0, 4, 1, 2, 3).reshape(N, cout, Ho, -1)
    return v, y.store


def _K(sig):
    prec, fn, cin, _, k = sig[:5]
    return 64 * k if fn == "stem" and prec != "fp32" else cin * k * k


def _reference(sig, ref, rows=None):
    """conv_grad_oracle.forward of the row on the device -> (want, bound, slack, c); rows=(h0, h1): output rows h0..h1
    only, from the input rows they read."""
    prec, fn, cin, cout, k, s, p, d, bias, relu, res, xin, out, pg, sf, ndev = sig
    x, w, b, r = ref
    pad = p
    if rows is not None:
        h0, h1 = rows
        lo, hi = s * h0, s * (h1 - 1) + d * (k - 1) + 1

        def band(t):
            return torch.nn.functional.pad(t, (0, 0, p, p))[:, :, lo:hi]
        x = tuple(band(t) for t in x) if isinstance(x, tuple) else band(x)
        r = None if r is None else r[:, :, h0:h1]
        pad = (0, p)
    want, bound, slack = CG.forward(x, w, b, s, pad, d, r, res == "up2", relu, prec, sf)
    c = CG.forward_c(prec, _K(sig), int(bias) + int(res is not None))
    st = CG.store_slack(want, bound, c, {"pair": "pair", "bf16": "bf16"}.get(out, "f32"))
    return want, bound, st if slack is None else st + slack, c


def _check(key, got, want, bound, slack, c):
    ok, ratio = G.check(got, want, bound, c, slack=slack)
    WORST[key] = (max(WORST.get(key, (0.0, c))[0], ratio), c)
    assert ok, "%s: worst err/bound %.3e > c %.3e" % (key, ratio, c)


def _tma_route(sig):
    """Whether launch_igemm_tma (csrc/igemm_tma.cu) takes the row: bf16 activations at precision bf16 or pairs at
    bf16x3 (fp32 rows at bf16x3 become pairs on entry), Cin % 64 == 0, stride 2 only for 1x1 / pad 0; an fp32, NCHW
    or Cout % 64 output takes the direct-store epilogue, which has no residual and at most 256 channels; the up2
    residual needs an even output."""
    prec, fn, cin, cout, k, s, p, d, bias, relu, res, xin, out, pg, sf, ndev = sig
    if prec == "fp32" or fn == "stem":
        return False
    if prec == "bf16" and xin != "bf16":
        return False
    direct = out not in ("pair", "bf16") or cout % 64 != 0
    return cin % 64 == 0 and not (direct and (res is not None or cout > 256)) and (s == 1 or (k == 1 and p == 0))


def _pair_like(sig):
    return sig[0] == "bf16x3"


def routes(sig):
    """[(route, kernel regex)] of the row: 'simt'; 'stem'; 'tma' (default N tile), 'tma64' (where Cout rounded up is a
    multiple of 64; a 32-channel head keeps its 32 tile), 'tma128' (where it is a multiple of 128 and the kernel keeps
    the tile) and 'gather' (ops.USE_TMA off: every TMA row but the pair-group deconv, which only the TMA kernel
    writes); 'gather' alone for the rows the TMA kernel does not take."""
    prec, fn, cin, cout = sig[:4]
    if prec == "fp32":
        return [("simt", r"igemm_simt_kernel")]
    if fn == "stem":
        return [("stem", r"stem_pack_image_kernel|igemm_tma_kernel<\d+, ?%d>" % (1 if prec == "bf16x3" else 0))]
    xm = 2 if _pair_like(sig) else (1 if sig[11] == "bf16" else 0)
    cp = 32 if cout <= 32 else (cout + 63) // 64 * 64
    gather = ("gather", r"igemm_tc_kernel<0, ?%d, ?%d>" % (xm, min(cp, 64)))
    if not _tma_route(sig):
        return [gather]
    mma = 1 if prec == "bf16x3" else 0

    def tma(bn):
        return r"igemm_tma_kernel<%s, ?%d>" % (r"\d+" if bn is None else (2 * bn if mma else bn), mma)
    out = [("tma", tma(None))]
    if cp % 64 == 0:
        out.append(("tma64", tma(64)))
    # the pair kernel narrows a 128 tile whose ring would get fewer than three stages to 64: beside a residual slab or
    # the direct epilogue's staging
    direct = sig[12] not in ("pair", "bf16") or cout % 64 != 0
    if cp % 128 == 0 and not (mma and (sig[10] is not None or direct)):
        out.append(("tma128", tma(128)))
    if not sig[13]:
        out.append(gather)
    return out


def _set_route(route):
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import lib
    assert lib().upsnet_tma_set_tile_n({"tma64": 64, "tma128": 128}.get(route, 0)) == 0
    ops.USE_TMA["on"] = route != "gather"


def run_row(U, monkeypatch, name, sig, size, seed, dev, route):
    U.set_precision(sig[0])
    _set_route(route)
    args, ref, (N, Ho, Wo) = _inputs(sig, size, seed, dev)
    with monkeypatch.context() as mp:
        seen = _record(mp)
        y = _call(sig, size, args)
    assert sig in seen, "%s: the call has the signature %s, not the row's" % (name, sorted(seen, key=repr))
    got, store = _got(y, sig)
    want, bound, slack, c = _reference(sig, ref)
    assert got.shape == want.shape, (got.shape, want.shape)
    n = N - 1 if sig[15] else N             # n_dev: only the images below the count are computed
    _check("%s [%s]" % (name, route), got[:n], want[:n], bound[:n], slack[:n], c)
    if store is not None:
        G.check_pair_split(store[:n])


@pytest.mark.parametrize("row", LAYERS, ids=[r[0] for r in LAYERS])
def test_layer(dev, engine, monkeypatch, row):
    name, sig, size = row
    if sig[5] == 2 and len(size) == 3:
        assert size[1] % 2 == 1, "stride-2 rows run at an odd H"
    for route, _ in routes(sig):
        run_row(engine, monkeypatch, name, sig, size, LAYERS.index(row), dev, route)


@pytest.mark.parametrize("prec", PRECS)
def test_routes(dev, engine, prec):
    """Each (row, route) launches the kernel instance routes() names, read from one profiler session per precision."""
    engine.set_precision(prec)
    calls, want = [], []
    for i, (name, sig, size) in enumerate(LAYERS):
        if sig[0] != prec:
            continue
        for route, kernel in routes(sig):
            args, _, _ = _inputs(sig, size, i, dev)

            def fn(sig=sig, size=size, args=args, route=route):
                _set_route(route)
                _call(sig, size, args)
            calls.append(fn)
            want.append((name, route, kernel))
    got = launched_kernels_each(calls, lambda n: "igemm" in n or "stem" in n)
    bad = []
    for (name, route, kernel), names in zip(want, got):
        pats = kernel.split("|")
        names = {n for n in names if "pack_weight" not in n}
        if not names or any(not any(re.search(p, n) for p in pats) for n in names) or \
                any(not any(re.search(p, n) for n in names) for p in pats):
            bad.append("%s [%s]: launched %s, want %s" % (name, route, sorted(names), kernel))
        print("conv forward route %-40s %-7s %s" % (name, route, sorted(names)))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------
# full size (bf16x3, the benchmark's tile choice)
# ------------------------------------------------------------------------------------------------
FULL = [
    # 1024 x 2048: res2 conv3 + residual and the FPN 3x3 at 256 x 512, res5 3x3 at 32 x 64, the stem, fc6 at 1000 rois
    ("full res2 conv3 +res", _sig("bf16x3", 64, 256, relu=True, res="same"), (1, 256, 512)),
    ("full fpn 3x3", _sig("bf16x3", 256, 256, 3, 1, 1), (1, 256, 512)),
    ("full res5 3x3", _sig("bf16x3", 512, 512, 3, 1, 1, relu=True), (1, 32, 64)),
    ("full stem", _sig("bf16x3", 3, 64, 7, 2, 3, relu=True, xin="f32 nchw", fn="stem"), (1, 1024, 2048)),
    ("full fc6", _sig("bf16x3", 12544, 1024, relu=True), (1000,)),
    # 800 x 1344: the FPN 3x3 at 200 x 336, res5 3x3 at 25 x 42
    ("full coco fpn 3x3", _sig("bf16x3", 256, 256, 3, 1, 1), (1, 200, 336)),
    ("full coco res5 3x3", _sig("bf16x3", 512, 512, 3, 1, 1, relu=True), (1, 25, 42)),
]


@pytest.mark.parametrize("row", FULL, ids=[r[0] for r in FULL])
def test_fullsize(dev, engine, row):
    name, sig, size = row
    engine.set_precision("bf16x3")
    args, ref, (N, Ho, Wo) = _inputs(sig, size, len(name), dev)
    got, store = _got(_call(sig, size, args), sig)
    bands = [(0, min(8, Ho))] + ([(Ho - 8, Ho)] if Ho > 16 else [])
    for h0, h1 in bands:
        want, bound, slack, c = _reference(sig, ref, (h0, h1))
        _check(name, got[:, :, h0:h1], want, bound, slack, c)
    if store is not None:
        G.check_pair_split(store)


def test_teeth(dev, engine):
    """A 3x3 pair row (256 -> 256) through upsnet_igemm_forward with one tap's 64-channel k-block zeroed in a copy of
    its packed weight: the check must fail (the intact weight passes)."""
    from upsnet_b200 import _lib
    from upsnet_b200 import operators as ops
    sig = _sig("bf16x3", 256, 256, 3, 1, 1, relu=True)
    engine.set_precision("bf16x3")
    args, ref, (N, Ho, Wo) = _inputs(sig, (1, 13, 22), 5, dev)
    x, w, b, _ = args
    packed = ops._packed_weight(w)
    Kp = 9 * 256
    results = []
    for zero in (False, True):
        p = packed.clone()
        if zero:
            planes = p.view(torch.bfloat16).view(2, -1, Kp)
            planes[:, :, 4 * 256 + 128:4 * 256 + 192] = 0          # tap 4 (the centre), channels 128..191
        store = torch.empty((N, Ho, Wo, 512), dtype=torch.bfloat16, device=dev)
        _lib.call("igemm_forward", dev, x.store, None, None, p, b, None, store, N, 13, 22, 256, 256, 3, 3, 1, 1, 1, 1,
                  1, 1, _lib.LAYOUT_NHWC, _lib.DTYPE_PAIR, _lib.DTYPE_PAIR, _lib.EPI_RELU, _lib.PREC_BF16X3, None)
        want, bound, slack, c = _reference(sig, ref)
        results.append(G.check(ops.Pair(store).float().double(), want, bound, c, slack=slack))
    assert results[0][0], results[0]
    assert not results[1][0], results[1]


# ------------------------------------------------------------------------------------------------
# census: every dense signature the inference forward calls is a row
# ------------------------------------------------------------------------------------------------
CONFIGS = {"cityscapes_r50": (256, 512), "coco_r50": (256, 384), "coco_r101_dcn": (256, 384)}


def _census(config, monkeypatch):
    """The dense signatures the inference forward of a synthetic model of the configuration (depth 2, 2, 2, 2: block 0
    and one later block per stage, which have all the signatures of the full depth) calls, in each precision."""
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    dev = torch.device("cuda", 0)
    H, W = CONFIGS[config]
    m = synthetic_model(getattr(UPSNetConfig, config)(), depth=(2, 2, 2, 2), seed=1, device=dev)
    m.use_cuda_graph = False
    inp = synthetic_input(H, W, seed=2, device=dev)
    seen = _record(monkeypatch)
    try:
        for prec in PRECS:
            U.set_precision(prec)
            with torch.no_grad():
                m(inp)
            torch.cuda.synchronize()
    finally:
        U.set_precision("fp32")
    return seen


_CHILD = """
import json, sys
sys.path[:0] = [%r, %r]
import pytest
import test_gpu_conv_forward_fp64 as T
with pytest.MonkeyPatch.context() as mp:
    print(json.dumps(sorted(T._census(%r, mp), key=repr)))
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_census(dev, config):
    """In a child process, as tests/test_gpu_conv_backward_wide.py's census: the model's forward is kept out of the
    test process, whose later profiler sessions would otherwise lose their records (tests/kernel_trace.py)."""
    import json
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    out = subprocess.run([sys.executable, "-s", "-c", _CHILD % (here, os.path.dirname(here), config)],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    seen = {tuple(s) for s in json.loads(out.stdout.strip().splitlines()[-1])}
    assert {s[0] for s in seen} == set(PRECS) and any(s[1] == "stem" for s in seen), sorted(seen, key=repr)
    missing = sorted(seen - {r[1] for r in LAYERS}, key=repr)
    assert not missing, "%s calls dense layers no row covers: %s" % (config, missing)
