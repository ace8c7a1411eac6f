"""GroupNorm on the device (csrc/group_norm.cu; network.*_with_norm = 'group_norm').

Kernels against float64 F.group_norm (and its autograd) at every GN layer shape of cityscapes_r50 (1024x2048) and
coco_r50 (800x1344), in the three storage formats, with ReLU, the nearest-2x residual and the extra shift; byte
repeatability and graph replay.  Whole-model inference with all norm keys 'group_norm' against the literal model
(oracle/literal_model.py), graphs over mixed sizes, and the training forward against the float64 oracle."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402
from oracle.literal_model import LiteralUPSNet  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
NORM_KEYS = ("fpn_with_norm", "rpn_with_norm", "rcnn_with_norm", "fcn_with_norm")
# worst error / sum of |terms| of the output: fp32 statistics of up to 2^25-element groups, plus the output rounding
STAT_TOL = 2e-5
OUT_TOL = {"f32": 2.0 ** -23, "pair": 2.0 ** -16, "bf16": 2.0 ** -8}


def _gn_cfg(base):
    for k in NORM_KEYS:
        setattr(base, k, "group_norm")
    return base


def _as(x, fmt):
    """logical fp32 [N,C,H,W] -> the activation format under test, and its exactly decoded fp32 value"""
    from upsnet_b200 import operators as ops
    if fmt == "pair":
        p = ops.Pair.from_float(x)
        return p, p.float()
    if fmt == "bf16":
        b = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        return b, b.float()
    f = x.contiguous(memory_format=torch.channels_last)
    return f, f


def _check(got, x, gamma, beta, fmt, relu=False, res=None, shift=None, rows=None):
    from upsnet_b200 import operators as ops
    got = ops.as_float(got).double()
    x, gamma, beta = x.double(), gamma.double(), beta.double()
    if x.dim() == 2:
        x, got = x[:, :, None, None], got.reshape(x.shape[0], -1, 1, 1)
    C = x.shape[1]
    xh = F.group_norm(x, 32, None, None, 1e-5)
    want = xh * gamma.view(1, C, 1, 1) + beta.view(1, C, 1, 1)
    # the terms of (x - mean) rstd gamma + beta: |x| and |mean| scaled by rstd |gamma|, and |beta|
    xg = x.reshape(x.shape[0], 32, -1)
    mean = xg.mean(-1, keepdim=True)
    rstd = 1 / (xg.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    scale = ((xg.abs() + mean.abs()) * rstd).reshape(x.shape)
    terms = scale * gamma.abs().view(1, C, 1, 1) + beta.abs().view(1, C, 1, 1)
    if shift is not None:
        want = want + shift.double()[:, :, None, None]
        terms = terms + shift.double().abs()[:, :, None, None]
    if res is not None:
        up = F.interpolate(ops.as_float(res).double(), scale_factor=2, mode="nearest")
        want, terms = want + up, terms + up.abs()
    if relu:
        want = want.clamp_min(0)
    if rows is not None:
        got, want, terms = got[:rows], want[:rows], terms[:rows]
    err = float(((got - want).abs() / (terms + 1e-30)).max())
    assert err <= STAT_TOL + OUT_TOL[fmt], (fmt, err)
    return err


MAP_SHAPES = [(256, 512, 256), (128, 256, 256), (64, 128, 256), (32, 64, 256), (16, 32, 256),       # FPN/RPN 1024x2048
              (200, 336, 256), (100, 168, 256), (50, 84, 256), (25, 42, 256), (13, 21, 256),        # 800x1344
              (256, 512, 128), (128, 256, 128), (64, 128, 128), (32, 64, 128),                       # FCN 1024x2048
              (200, 336, 128), (25, 42, 128)]
OPTIONS = ["plain", "relu", "res", "shift_res"]


def _run_map(H, W, C, fmt, opt, seed):
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(seed)
    x32 = (torch.randn(1, C, H, W, generator=g) * 3 + 5).to(DEV)     # an offset mean: the statistics must not cancel
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.1).to(DEV)
    x, xv = _as(x32, fmt)
    kw = {"relu": opt == "relu"}
    res = shift = None
    if opt in ("res", "shift_res") and H % 2 == 0 and W % 2 == 0:
        res, _ = _as(torch.randn(1, C, H // 2, W // 2, generator=g).to(DEV), fmt)
        kw.update(residual=res, residual_up2=True)
    if opt == "shift_res":
        shift = torch.randn(1, C, generator=g).to(DEV)
        kw["shift"] = shift
    y = ops.group_norm(x, gamma, beta, **kw)
    assert type(y) is type(x) and tuple(y.shape) == (1, C, H, W)
    err = _check(y, xv, gamma, beta, fmt, kw["relu"], res, shift)
    again = ops.group_norm(x, gamma, beta, **kw)
    assert torch.equal(_store(y), _store(again))
    return err


def _store(y):
    from upsnet_b200 import operators as ops
    return y.store if isinstance(y, ops.Pair) else y


@pytest.mark.parametrize("fmt", ["pair", "bf16", "f32"])
@pytest.mark.parametrize("i", range(len(MAP_SHAPES)))
def test_map_group_norm_vs_fp64(fmt, i):
    H, W, C = MAP_SHAPES[i]
    _run_map(H, W, C, fmt, OPTIONS[i % 4], seed=i)


@pytest.mark.parametrize("fmt", ["pair", "bf16", "f32"])
@pytest.mark.parametrize("opt", OPTIONS)
def test_map_group_norm_options(fmt, opt):
    _run_map(64, 128, 256, fmt, opt, seed=100)


@pytest.mark.parametrize("fmt", ["pair", "bf16", "f32"])
@pytest.mark.parametrize("R", [1, 100, 128])
def test_rows_mask_branch(fmt, R):
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(R)
    x32 = (torch.randn(R, 256, 14, 14, generator=g) * 2 + 1).to(DEV)
    gamma = (torch.rand(256, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(256, generator=g) * 0.1).to(DEV)
    x, xv = _as(x32, fmt)
    y = ops.group_norm_rows(x, gamma, beta, relu=True)
    _check(y, xv, gamma, beta, fmt, relu=True)
    n = max(1, R - 37)
    y2 = ops.group_norm_rows(x, gamma, beta, relu=True, n_dev=torch.tensor([n], dtype=torch.int32, device=DEV))
    _check(y2, xv, gamma, beta, fmt, relu=True, rows=n)
    assert torch.equal(_store(y)[:n], _store(y2)[:n])


@pytest.mark.parametrize("fmt", ["pair", "bf16", "f32"])
@pytest.mark.parametrize("R", [1, 512, 1000])
def test_rows_fc6(fmt, R):
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(R + 7)
    x32 = (torch.randn(R, 1024, generator=g) * 4).to(DEV)
    gamma = (torch.rand(1024, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(1024, generator=g) * 0.1).to(DEV)
    if fmt == "pair":      # the engine's pair-stream fc6 output: R one-pixel images
        x = ops.Pair.from_float(x32[:, :, None, None])
        xv = x.float().reshape(R, 1024)
    else:
        x = x32.to(torch.bfloat16) if fmt == "bf16" else x32
        xv = x.float()
    y = ops.group_norm_rows(x, gamma, beta, relu=True)
    _check(y, xv, gamma, beta, fmt, relu=True)


def test_graph_replay_is_byte_identical():
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(5)
    x, _ = _as(torch.randn(1, 256, 128, 256, generator=g).to(DEV), "pair")
    res, _ = _as(torch.randn(1, 256, 64, 128, generator=g).to(DEV), "pair")
    r, _ = _as(torch.randn(100, 256, 14, 14, generator=g).to(DEV), "pair")
    gamma, beta = torch.rand(256, generator=g).to(DEV) + 0.5, torch.randn(256, generator=g).to(DEV)
    shift = torch.randn(1, 256, generator=g).to(DEV)
    n = torch.tensor([60], dtype=torch.int32, device=DEV)

    def run():
        return (ops.group_norm(x, gamma, beta, residual=res, residual_up2=True, shift=shift).store,
                ops.group_norm_rows(r, gamma, beta, relu=True, n_dev=n).store)
    eager = [t.clone() for t in run()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], eager[0])
        assert torch.equal(out[1][:60], eager[1][:60])


@pytest.mark.parametrize("N,H,W,C,relu,res,shift", [
    (1, 128, 256, 256, False, True, False),      # FPN lateral with the top-down add
    (1, 25, 42, 256, False, False, True),        # P5 lateral with the context vector (odd sizes)
    (1, 64, 128, 128, True, False, False),       # FCN layer
    (64, 14, 14, 256, True, False, False),       # mask rows
    (512, 1, 1, 1024, True, False, False),       # fc6 rows
])
def test_backward_vs_fp64_autograd(N, H, W, C, relu, res, shift):
    from upsnet_b200 import training
    g = torch.Generator().manual_seed(N * H + C)
    x = (torch.randn(N, C, H, W, generator=g) * 2 + 3).to(DEV).contiguous(memory_format=torch.channels_last)
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.1).to(DEV)
    r = torch.randn(N, C, H // 2, W // 2, generator=g).to(DEV) if res else None
    sh = torch.randn(N, C, generator=g).to(DEV) if shift else None
    dy = torch.randn(N, C, H, W, generator=g).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in (x, gamma, beta)]
    extra = [None if t is None else t.clone().requires_grad_(True) for t in (r, sh)]
    y = training.group_norm(leaves[0], leaves[1], leaves[2], relu=relu, residual=extra[0], shift=extra[1])
    y.backward(dy)
    d = [t.double().detach().requires_grad_(True) for t in (x, gamma, beta)]
    de = [None if t is None else t.double().detach().requires_grad_(True) for t in (r, sh)]
    w = F.group_norm(d[0], 32, d[1], d[2], 1e-5)
    if de[1] is not None:
        w = w + de[1][:, :, None, None]
    if de[0] is not None:
        w = w + F.interpolate(de[0], scale_factor=2, mode="nearest")
    if relu:
        w = w.clamp_min(0)
    assert float((y.detach().double() - w.detach()).abs().max()) <= 1e-4 * float(w.detach().abs().max())
    w.backward(dy.double())
    for a, b in zip(leaves + [e for e in extra if e is not None], d + [e for e in de if e is not None]):
        rel = float((a.grad.double() - b.grad).norm() / b.grad.norm())
        assert rel <= 1e-4, rel
    again = training.group_norm(x.clone().requires_grad_(True), gamma, beta, relu=relu, residual=r, shift=sh)
    assert torch.equal(again, y.detach())


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return ((a - b).abs().max() / max(1.0, float(b.abs().max()))).item()


@pytest.mark.parametrize("name,H,W", [("cityscapes_r50", 1024, 2048), ("coco_r50", 800, 1344)])
def test_model_inference_vs_literal(name, H, W):
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    depth = (3, 4, 6, 3)
    cfg = _gn_cfg(getattr(UPSNetConfig, name)())
    m = synthetic_model(cfg, depth=depth, seed=0, device=DEV)
    m.keep_intermediates = True
    inp = synthetic_input(H, W, seed=3, device=DEV)
    U.set_precision("bf16x3")
    try:
        with torch.no_grad():
            out = m(inp)
    finally:
        U.set_precision("fp32")
        m.keep_intermediates = False
    it = out["_intermediates"]
    lit = LiteralUPSNet(m.state_dict(), depth=depth, num_classes=cfg.num_classes, num_seg_classes=cfg.num_seg_classes,
                        dconv_from=cfg.backbone_with_dconv, fcn_layers=cfg.fcn_num_layers, with_gap=cfg.fpn_with_gap,
                        dtype=torch.float64, device=DEV)
    d = lit.dense(inp["data"])
    errs = {"fpn_p%d" % (l + 2): rel(a, b) for l, (a, b) in enumerate(zip(it["fpn"], d["fpn"]))}
    for l in range(5):
        errs["rpn_prob%d" % l] = rel(it["rpn_cls_prob"][l], d["rpn"][l][2])
        errs["rpn_bbox%d" % l] = rel(it["rpn_bbox_pred"][l], d["rpn"][l][1])
    errs["fcn_output"] = rel(it["fcn_output"], d["fcn_output"])
    feats = list(d["fpn"][:4])
    valid = it["roi_valid"]
    rois = it["rois"][valid]
    with torch.no_grad():
        r = lit.rcnn(feats, rois)
        errs["cls_score"] = rel(it["cls_score"][valid], r["cls_score"])
        errs["bbox_pred"] = rel(it["bbox_pred"][valid], r["bbox_pred"])
        n1 = out["pred_boxes"].shape[0]
        if n1:
            errs["mask_probs"] = rel(out["mask_probs"], torch.sigmoid(lit.mask_branch(feats, out["pred_boxes"])))
    print("%s group_norm max rel errors:" % name, {k: "%.2e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if v > 1e-3}
    assert not bad, bad
    assert n1 > 0


def test_model_graphs_over_mixed_sizes():
    """Two padded shapes through captured graphs (A, B, A) equal the eager static forward of each, bit for bit."""
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    m = synthetic_model(_gn_cfg(UPSNetConfig.coco_r50()), depth=(1, 1, 1, 1), seed=3, device=DEV)
    imgs = [synthetic_input(h, w, seed=40 + i, device=DEV) for i, (h, w) in enumerate([(128, 192), (96, 160)])]
    U.set_precision("bf16x3")
    try:
        with torch.no_grad():
            m.use_cuda_graph = False
            want = [{k: v.clone() for k, v in m(x).items() if torch.is_tensor(v)} for x in imgs]
            m.use_cuda_graph = True
            m._graphs = {}
            for j in (0, 1, 0):
                got = {k: v for k, v in m(imgs[j]).items() if torch.is_tensor(v)}
                for k in want[j]:
                    assert torch.equal(got[k], want[j][k]), k
            assert len(m._graphs) == 2
    finally:
        U.set_precision("fp32")
        m.use_cuda_graph = True


def test_pipelined_engine_mixed_sizes():
    """PipelinedEngine over raw images of mixed sizes with group_norm heads == one engine per image geometry."""
    import upsnet_b200 as U
    import train_sample_cases as TS
    from upsnet_b200.geometry import image_geometry
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    m = synthetic_model(_gn_cfg(UPSNetConfig.cityscapes_r50()), depth=(1, 1, 1, 1), seed=3, device=DEV)
    small = (96, 160)
    sizes = [(64, 90), (81, 64), (60, 200)]
    raws = [torch.from_numpy(TS.image_bgr(h, w, 90 + i)).pin_memory() for i, (h, w) in enumerate(sizes)]
    U.set_precision("bf16x3")
    try:
        eng = U.PipelinedEngine(m, depth=4, lanes=2, target_size=small[0], max_size=small[1], max_image_shape=(120, 200))
        tickets = [eng.submit(r) for r in raws]
        got = [{k: v.clone() for k, v in eng.result(t).items()} for t in tickets]
        for i, r in enumerate(raws):
            g = image_geometry(*sizes[i], *small)
            ref = U.PipelinedEngine(m, g.im_info[None], depth=2, im_scale=g.scale)
            want = ref.result(ref.submit(r))
            assert got[i].keys() == want.keys()
            for k in want:
                if torch.is_tensor(want[k]):
                    assert torch.equal(got[i][k], want[k]), (i, k)
    finally:
        U.set_precision("fp32")


# ------------------------------------------------------------------------------------------------
# training forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_gap", [False, True])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_training_forward_vs_oracle(prec, with_gap):
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    from upsnet_b200.training import PanopticLabels, RPNTargets
    depth, H, W, seed = (2, 2, 2, 2), 256, 512, 0
    cfg = _gn_cfg(UPSNetConfig(fpn_with_gap=with_gap))
    m = synthetic_model(cfg, depth=depth, seed=seed, device=DEV)
    entry, lmap = TF.synthetic_entry(seed + 1, H, W, 8)
    label = {"roidb": entry}
    np.random.seed(seed)
    label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, DEV))
    label.update(PanopticLabels(dataset="cityscapes").from_roidb(entry, lmap, (H, W), 1.0, DEV))
    data = {"data": TF.image(seed + 2, H, W).to(DEV), "im_info": np.array([[H, W, 1.0]], np.float32)}
    saved = ops._PRECISION["conv"]
    U.set_precision(prec)
    try:
        m.keep_intermediates = True
        m.zero_grad(set_to_none=True)
        np.random.seed(5)
        out = m(data, label)
        sum(out[k] for k in TF.LOSSES).backward()
    finally:
        ops._PRECISION["conv"] = saved
    trainable = set(TF.trainable_names(m))
    assert any(".fc6.2." in k for k in trainable) and any("fpn_p2.1." in k for k in trainable)
    for k, p in m.named_parameters():
        assert (p.grad is not None) == (k in trainable), k
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    orc = TF.TrainOracle(sd, TF.trainable_names(m), depth=depth, with_gap=with_gap, dtype=torch.float64, device=DEV)
    want, wgrads = orc.step(data["data"], label, out["_intermediates"])
    named = dict(m.named_parameters())
    got = {k: named[k].grad for k in wgrads}
    err = TF.grad_errors(got, wgrads)
    worst = max(err, key=err.get)
    print("\n[group_norm %s gap=%s] worst grad rel L2 %.3e (%s)" % (prec, with_gap, err[worst], worst))
    bad = {k: e for k, e in err.items() if e > TF.grad_tol(k, prec)}
    assert not bad, bad
    for k in TF.LOSSES:
        assert abs(float(out[k]) - want[k]) / max(abs(want[k]), 1e-3) <= TF.LOSS_TOL[prec], k
