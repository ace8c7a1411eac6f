"""The FPN's bilinear top-down path on the device (network.fpn_upsample_method = 'bilinear'; csrc/upsample2.cu and the
GroupNorm apply's bilinear residual mode in csrc/group_norm.cu).

Kernels against float64 F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) and its autograd, at every
FPN level shape of cityscapes_r50 (1024x2048) and coco_r50 (800x1344) and at odd sizes, in the three storage formats;
the GroupNorm apply's bilinear mode and its backward against float64 F.group_norm + F.interpolate; byte repeatability
and graph replay.  Whole-model inference with 'bilinear' for both norms against the literal model
(tests/fpn_upsample_oracle.py: oracle/literal_model.py with the bilinear FPN), in all three precisions, graphs over mixed sizes, PipelinedEngine,
and the training forward against the float64 oracle."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402
from fpn_upsample_oracle import BilinearLiteralUPSNet, BilinearTrainOracle  # noqa: E402
from oracle.literal_model import LiteralUPSNet  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
NORM_KEYS = ("fpn_with_norm", "rpn_with_norm", "rcnn_with_norm", "fcn_with_norm")
# worst error / interpolation of |x| (the sum of the |terms|): fp32 blend (a few ulps) plus the output rounding
OUT_TOL = {"f32": 2.0 ** -23, "pair": 2.0 ** -16, "bf16": 2.0 ** -8}
BLEND_TOL = 4 * 2.0 ** -24
STAT_TOL = 2e-5


def _up(x):
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)


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


def _store(y):
    from upsnet_b200 import operators as ops
    return y.store if isinstance(y, ops.Pair) else y


# coarse (h, w) of the three top-down up-samplings: P5->P4, P4->P3, P3->P2 of 1024x2048 and of 800x1344, and odd sizes
COARSE = [(32, 64), (64, 128), (128, 256), (25, 42), (50, 84), (100, 168), (3, 5), (1, 1), (1, 7), (13, 21)]


@pytest.mark.parametrize("fmt", ["pair", "bf16", "f32"])
@pytest.mark.parametrize("h,w", COARSE)
def test_upsample_forward_vs_fp64(fmt, h, w):
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(h * 1000 + w)
    x, xv = _as((torch.randn(1, 256, h, w, generator=g) * 3 + 1).to(DEV), fmt)
    y = ops.upsample2_bilinear(x)
    assert type(y) is type(x) and tuple(y.shape) == (1, 256, 2 * h, 2 * w)
    want, terms = _up(xv.double()), _up(xv.double().abs())
    err = float(((ops.as_float(y).double() - want).abs() / (terms + 1e-30)).max())
    assert err <= OUT_TOL[fmt] + BLEND_TOL, (fmt, err)
    assert torch.equal(_store(y), _store(ops.upsample2_bilinear(x)))


def test_upsample_forward_two_images_and_nchw_input():
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 64, 7, 9, generator=g).to(DEV)            # NCHW-contiguous fp32: copied to NHWC storage
    y = ops.upsample2_bilinear(x)
    assert float((y.double() - _up(x.double())).abs().max()) <= 1e-5 * float(x.abs().max())


@pytest.mark.parametrize("h,w", COARSE)
def test_adjoint_vs_fp64_autograd(h, w):
    from upsnet_b200 import training
    g = torch.Generator().manual_seed(h * 7 + w)
    dy = torch.randn(1, 256, 2 * h, 2 * w, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
    got = training.upsample2_bilinear_adjoint(dy)
    x = torch.zeros(1, 256, h, w, dtype=torch.float64, device=DEV, requires_grad=True)
    _up(x).backward(dy.double())
    xa = torch.zeros_like(x, requires_grad=True)
    _up(xa).backward(dy.double().abs())
    err = float(((got.double() - x.grad).abs() / (xa.grad + 1e-30)).max())
    assert err <= 8 * 2.0 ** -24, err
    assert torch.equal(got, training.upsample2_bilinear_adjoint(dy))


def test_autograd_function_forward_and_backward():
    from upsnet_b200 import training
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(1, 128, 25, 42, generator=g)).to(DEV).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(1, 128, 50, 84, generator=g).to(DEV)
    a = x.clone().requires_grad_(True)
    y = training.upsample2_bilinear(a)
    y.backward(dy)
    b = x.double().requires_grad_(True)
    w = _up(b)
    w.backward(dy.double())
    assert float((y.detach().double() - w.detach()).abs().max()) <= 1e-6 * float(w.detach().abs().max())
    assert float((a.grad.double() - b.grad).norm() / b.grad.norm()) <= 1e-6


# ------------------------------------------------------------------------------------------------
# GroupNorm apply with the bilinear residual
# ------------------------------------------------------------------------------------------------
def _gn_check(got, x, gamma, beta, fmt, res, relu=False, shift=None):
    from upsnet_b200 import operators as ops
    got = ops.as_float(got).double()
    x, gamma, beta = x.double(), gamma.double(), beta.double()
    C = x.shape[1]
    want = F.group_norm(x, 32, None, None, 1e-5) * gamma.view(1, C, 1, 1) + beta.view(1, C, 1, 1)
    xg = x.reshape(x.shape[0], 32, -1)
    mean = xg.mean(-1, keepdim=True)
    rstd = 1 / (xg.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    terms = ((xg.abs() + mean.abs()) * rstd).reshape(x.shape) * gamma.abs().view(1, C, 1, 1) + beta.abs().view(1, C, 1, 1)
    if shift is not None:
        want, terms = want + shift.double()[:, :, None, None], terms + shift.double().abs()[:, :, None, None]
    r = ops.as_float(res).double()
    want, terms = want + _up(r), terms + _up(r.abs())
    if relu:
        want = want.clamp_min(0)
    err = float(((got - want).abs() / (terms + 1e-30)).max())
    assert err <= STAT_TOL + OUT_TOL[fmt], (fmt, err)
    return err


# fine (H, W) of the GN'd FPN laterals with a top-down residual: P4, P3, P2 of 1024x2048 and of 800x1344, and odd P5
GN_FINE = [(64, 128), (128, 256), (256, 512), (50, 84), (100, 168), (200, 336), (6, 10)]


@pytest.mark.parametrize("fmt", ["pair", "bf16", "f32"])
@pytest.mark.parametrize("H,W", GN_FINE)
def test_group_norm_bilinear_residual_vs_fp64(fmt, H, W):
    from upsnet_b200 import operators as ops
    g = torch.Generator().manual_seed(H + W)
    x, xv = _as((torch.randn(1, 256, H, W, generator=g) * 3 + 5).to(DEV), fmt)
    gamma = (torch.rand(256, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(256, generator=g) * 0.1).to(DEV)
    res, _ = _as(torch.randn(1, 256, H // 2, W // 2, generator=g).to(DEV), fmt)
    shift = torch.randn(1, 256, generator=g).to(DEV) if H % 3 == 0 else None
    y = ops.group_norm(x, gamma, beta, residual=res, residual_up2=True, shift=shift, upsample="bilinear")
    assert type(y) is type(x) and tuple(y.shape) == (1, 256, H, W)
    _gn_check(y, xv, gamma, beta, fmt, res, shift=shift)
    assert torch.equal(_store(y), _store(ops.group_norm(x, gamma, beta, residual=res, residual_up2=True, shift=shift,
                                                        upsample="bilinear")))
    near = ops.group_norm(x, gamma, beta, residual=res, residual_up2=True, shift=shift)
    assert not torch.equal(_store(near), _store(y))


def test_group_norm_bilinear_relu_and_bad_keyword():
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import UpsnetError
    g = torch.Generator().manual_seed(8)
    x, xv = _as(torch.randn(2, 128, 50, 84, generator=g).to(DEV), "pair")
    gamma, beta = (torch.rand(128, generator=g) + 0.5).to(DEV), torch.randn(128, generator=g).to(DEV)
    res, _ = _as(torch.randn(2, 128, 25, 42, generator=g).to(DEV), "pair")
    y = ops.group_norm(x, gamma, beta, relu=True, residual=res, residual_up2=True, upsample="bilinear")
    _gn_check(y, xv, gamma, beta, "pair", res, relu=True)
    with pytest.raises(UpsnetError, match="upsample"):
        ops.group_norm(x, gamma, beta, residual=res, residual_up2=True, upsample="bicubic")


@pytest.mark.parametrize("N,H,W,C,relu,shift", [
    (1, 128, 256, 256, False, False),      # FPN P3 lateral of 1024x2048
    (1, 50, 84, 256, False, True),         # P4 lateral of 800x1344 (its residual P5 is 25x42)
    (1, 6, 10, 256, True, False),          # odd 3x5 residual, with the ReLU mask
    (2, 32, 64, 128, False, True),
])
def test_group_norm_bilinear_backward_vs_fp64_autograd(N, H, W, C, relu, shift):
    from upsnet_b200 import training
    g = torch.Generator().manual_seed(N * H + C)
    x = (torch.randn(N, C, H, W, generator=g) * 2 + 3).to(DEV).contiguous(memory_format=torch.channels_last)
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.1).to(DEV)
    r = torch.randn(N, C, H // 2, W // 2, generator=g).to(DEV)
    sh = torch.randn(N, C, generator=g).to(DEV) if shift else None
    dy = torch.randn(N, C, H, W, generator=g).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in (x, gamma, beta, r)]
    xs = None if sh is None else sh.clone().requires_grad_(True)
    y = training.group_norm(leaves[0], leaves[1], leaves[2], relu=relu, residual=leaves[3], shift=xs,
                            upsample="bilinear")
    y.backward(dy)
    d = [t.double().detach().requires_grad_(True) for t in (x, gamma, beta, r)]
    ds = None if sh is None else sh.double().detach().requires_grad_(True)
    w = F.group_norm(d[0], 32, d[1], d[2], 1e-5) + _up(d[3])
    if ds is not None:
        w = w + ds[:, :, None, None]
    if relu:
        w = w.clamp_min(0)
    assert float((y.detach().double() - w.detach()).abs().max()) <= 1e-4 * float(w.detach().abs().max())
    w.backward(dy.double())
    pairs = list(zip(leaves, d)) + ([] if ds is None else [(xs, ds)])
    for a, b in pairs:
        rel = float((a.grad.double() - b.grad).norm() / b.grad.norm())
        assert rel <= 1e-4, rel
    again = [t.clone().requires_grad_(True) for t in (x, gamma, beta, r)]
    y2 = training.group_norm(again[0], again[1], again[2], relu=relu, residual=again[3], shift=sh, upsample="bilinear")
    y2.backward(dy)
    assert torch.equal(y2.detach(), y.detach()) and torch.equal(again[3].grad, leaves[3].grad)


def test_graph_replay_is_byte_identical():
    from upsnet_b200 import operators as ops, training
    g = torch.Generator().manual_seed(5)
    x, _ = _as(torch.randn(1, 256, 128, 256, generator=g).to(DEV), "pair")
    c, _ = _as(torch.randn(1, 256, 25, 42, generator=g).to(DEV), "pair")
    res, _ = _as(torch.randn(1, 256, 64, 128, generator=g).to(DEV), "pair")
    dy = torch.randn(1, 256, 50, 84, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
    gamma, beta = torch.rand(256, generator=g).to(DEV) + 0.5, torch.randn(256, generator=g).to(DEV)

    def run():
        return (ops.upsample2_bilinear(c).store, training.upsample2_bilinear_adjoint(dy),
                ops.group_norm(x, gamma, beta, residual=res, residual_up2=True, upsample="bilinear").store)
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
        for a, b in zip(out, eager):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _cfg(base, norm):
    base.fpn_upsample_method = "bilinear"
    for k in NORM_KEYS:
        setattr(base, k, norm)
    return base


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return ((a - b).abs().max() / max(1.0, float(b.abs().max()))).item()


def _calibrate_gap(m, x):
    """fpn_gap scaled so that its context vector has RMS 1 on the test image, as the synthetic laterals have (with the
    reference's nn.Linear init it dominates P5 and saturates the heads' logits, see test_gpu_train_forward_coco.py)."""
    with torch.no_grad():
        r5 = m.resnet_backbone.forward_train(x, "bf16x3")[3]
        g = TF.gap_vector(r5, m.fpn.fpn_gap.weight, m.fpn.fpn_gap.bias)
        s = 1.0 / float(g.pow(2).mean().sqrt())
        m.fpn.fpn_gap.weight.mul_(s)
        m.fpn.fpn_gap.bias.mul_(s)


def _literal(m, cfg, depth, upsample="bilinear"):
    cls = BilinearLiteralUPSNet if upsample == "bilinear" else LiteralUPSNet
    return cls(m.state_dict(), depth=depth, num_classes=cfg.num_classes, num_seg_classes=cfg.num_seg_classes,
               dconv_from=cfg.backbone_with_dconv, fcn_layers=cfg.fcn_num_layers, with_gap=cfg.fpn_with_gap,
               dtype=torch.float64, device=DEV)


@pytest.mark.parametrize("norm", ["none", "group_norm"])
@pytest.mark.parametrize("name,H,W", [("cityscapes_r50", 1024, 2048), ("coco_r50", 800, 1344)])
def test_model_inference_vs_literal(name, H, W, norm):
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    depth = (3, 4, 6, 3)
    cfg = _cfg(getattr(UPSNetConfig, name)(), norm)
    m = synthetic_model(cfg, depth=depth, seed=0, device=DEV)
    m.keep_intermediates = True
    inp = synthetic_input(H, W, seed=3, device=DEV)
    if cfg.fpn_with_gap:
        _calibrate_gap(m, inp["data"])
    U.set_precision("bf16x3")
    try:
        with torch.no_grad():
            out = m(inp)
    finally:
        U.set_precision("fp32")
        m.keep_intermediates = False
    it = out["_intermediates"]
    lit = _literal(m, cfg, depth)
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
    worst = max(errs, key=errs.get)
    print("\n%s %s bilinear max rel errors (worst %s %.2e):" % (name, norm, worst, errs[worst]),
          {k: "%.2e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if v > 1e-3}
    assert not bad, bad
    assert n1 > 0
    # the engine follows the bilinear graph: it is nearer to it than to the nearest-neighbour one
    near = _literal(m, cfg, depth, "nearest").fpn(*d["res"])
    assert rel(it["fpn"][0], near[0]) > 2 * errs["fpn_p2"]


@pytest.mark.parametrize("norm", ["none", "group_norm"])
@pytest.mark.parametrize("prec,tol", [("fp32", 1e-4), ("bf16x3", 1e-3), ("bf16", 5e-2)])
def test_fpn_levels_every_precision(prec, tol, norm):
    """The captured engine's FPN levels with 'bilinear' in each precision against the literal model (a small net)."""
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    depth = (1, 1, 1, 1)
    cfg = _cfg(UPSNetConfig.coco_r50(), norm)
    m = synthetic_model(cfg, depth=depth, seed=2, device=DEV)
    m.keep_intermediates = True
    inp = synthetic_input(224, 352, seed=4, device=DEV)     # P5 7x11
    U.set_precision(prec)
    try:
        with torch.no_grad():
            it = m(inp)["_intermediates"]
    finally:
        U.set_precision("fp32")
        m.keep_intermediates = False
    d = _literal(m, cfg, depth).dense(inp["data"])
    errs = [rel(a, b) for a, b in zip(it["fpn"], d["fpn"])]
    print("\n%s %s fpn max rel errors:" % (prec, norm), ["%.2e" % e for e in errs])
    assert max(errs) <= tol, errs


@pytest.mark.parametrize("norm", ["none", "group_norm"])
def test_model_graphs_over_mixed_sizes(norm):
    """Two padded shapes through captured graphs (A, B, A) equal the eager static forward of each, bit for bit."""
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    m = synthetic_model(_cfg(UPSNetConfig.coco_r50(), norm), depth=(1, 1, 1, 1), seed=3, device=DEV)
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


@pytest.mark.parametrize("norm", ["none", "group_norm"])
def test_pipelined_engine_mixed_sizes(norm):
    """PipelinedEngine over raw images of mixed sizes with the bilinear FPN == one engine per image geometry."""
    import upsnet_b200 as U
    import train_sample_cases as TS
    from upsnet_b200.geometry import image_geometry
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    m = synthetic_model(_cfg(UPSNetConfig.cityscapes_r50(), norm), depth=(1, 1, 1, 1), seed=3, device=DEV)
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
@pytest.mark.parametrize("norm", ["none", "group_norm"])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_training_forward_vs_oracle(prec, norm, with_gap):
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    from upsnet_b200.training import PanopticLabels, RPNTargets
    depth, H, W, seed = (2, 2, 2, 2), 256, 512, 0
    cfg = _cfg(UPSNetConfig(fpn_with_gap=with_gap), norm)
    m = synthetic_model(cfg, depth=depth, seed=seed, device=DEV)
    entry, lmap = TF.synthetic_entry(seed + 1, H, W, 8)
    label = {"roidb": entry}
    np.random.seed(seed)
    label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, DEV))
    label.update(PanopticLabels(dataset="cityscapes").from_roidb(entry, lmap, (H, W), 1.0, DEV))
    data = {"data": TF.image(seed + 2, H, W).to(DEV), "im_info": np.array([[H, W, 1.0]], np.float32)}
    if with_gap:
        _calibrate_gap(m, data["data"])
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
    for k, p in m.named_parameters():
        assert (p.grad is not None) == (k in trainable), k
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    orc = BilinearTrainOracle(sd, TF.trainable_names(m), depth=depth, with_gap=with_gap, dtype=torch.float64,
                              device=DEV)
    want, wgrads = orc.step(data["data"], label, out["_intermediates"])
    named = dict(m.named_parameters())
    got = {k: named[k].grad for k in wgrads}
    err = TF.grad_errors(got, wgrads)
    worst = max(err, key=err.get)
    print("\n[bilinear %s %s gap=%s] worst grad rel L2 %.3e (%s)" % (norm, prec, with_gap, err[worst], worst))
    bad = {k: e for k, e in err.items() if e > TF.grad_tol(k, prec)}
    assert not bad, bad
    for k in TF.LOSSES:
        assert abs(float(out[k]) - want[k]) / max(abs(want[k]), 1e-3) <= TF.LOSS_TOL[prec], k
