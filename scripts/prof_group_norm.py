"""GroupNorm cost: python scripts/prof_group_norm.py [iters]

1. Each GN pass (ops.group_norm: statistics + merge + apply, three launches; ops.group_norm_rows: one launch) at every
   GN layer shape of cityscapes_r50 (1024x2048) and coco_r50 (800x1344) with all *_with_norm = 'group_norm', in the pair
   (bf16x3) and bf16 streams: CUDA-event time per call over `iters` calls, the bytes the pass must move (statistics
   read + apply read + write, + the residual read where the FPN adds one), GB/s and the fraction of the H100 SXM's
   3.35 TB/s.  The FPN/RPN layers (one RPN conv per level is not normed, as in the reference) and the FCN layers count
   each shape as many times as the model runs it.
2. Engine images/s (the static forward replayed from its CUDA graph, host clock around `iters` replays ending in a
   synchronise) for both configurations with 'none' and with 'group_norm', bf16x3 and bf16.
3. One training step (forward(data, label) + backward, bf16x3) of cityscapes_r50 at 512x1024, 'none' and 'group_norm'.
The card, its power limit and clocks are read in the same run."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import upsnet_b200 as U  # noqa: E402
from prof_rpn_targets import card  # noqa: E402
from upsnet_b200 import operators as ops  # noqa: E402
from upsnet_b200.model import UPSNetConfig  # noqa: E402
from upsnet_b200.synthetic import synthetic_input, synthetic_model  # noqa: E402

HBM = 3.35e12
NORM_KEYS = ("fpn_with_norm", "rpn_with_norm", "rcnn_with_norm", "fcn_with_norm")
DEV = torch.device("cuda", 0)


def events_ms(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def layer_shapes(H, W, fcn_layers):
    """(name, kind, C, h, w, count, residual): the GN layers of the model at a padded H x W input."""
    out = []
    for l in range(2, 6):
        h, w = H >> l, W >> l
        out.append(("fpn_p%d_1x1" % l, "map", 256, h, w, 1, l < 5))
        out.append(("fpn_p%d" % l, "map", 256, h, w, 1, False))
        out.append(("fcn_p%d" % l, "map", 128, h, w, fcn_layers, False))
    out.append(("mask_conv x4 (100 rois)", "rows", 256, 14, 14, 4, False))
    out.append(("rcnn_fc6 (1000 rois)", "rows", 1024, 1, 1, 1, False))
    return out


def pass_table(iters):
    rows = []
    g = torch.Generator().manual_seed(0)
    for cfg_name, (H, W), fcn_layers in (("cityscapes_r50", (1024, 2048), 2), ("coco_r50", (800, 1344), 3)):
        for stream in ("pair", "bf16"):
            for name, kind, C, h, w, count, res in layer_shapes(H, W, fcn_layers):
                n = 1 if kind == "map" else (100 if C == 256 else 1000)
                x32 = torch.randn(n, C, h, w, generator=g).to(DEV)
                gamma, beta = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
                x = ops.Pair.from_float(x32) if stream == "pair" else x32.to(torch.bfloat16).contiguous(
                    memory_format=torch.channels_last)
                esize = 4 if stream == "pair" else 2
                nbytes = 3 * x32.numel() * esize
                kw = {}
                if kind == "map" and res:
                    r32 = torch.randn(1, C, h // 2, w // 2, generator=g).to(DEV)
                    kw = {"residual": ops.Pair.from_float(r32) if stream == "pair" else r32.to(torch.bfloat16),
                          "residual_up2": True}
                    nbytes += r32.numel() * esize
                if kind == "map":
                    fn = lambda: ops.group_norm(x, gamma, beta, **kw)          # noqa: E731
                else:
                    nbytes = 2 * x32.numel() * esize
                    xr = x if C == 256 else (x if stream == "pair" else x32.reshape(n, C).to(torch.bfloat16))
                    fn = lambda: ops.group_norm_rows(xr, gamma, beta, relu=True)   # noqa: E731
                ms = events_ms(fn, iters)
                rows.append({"config": cfg_name, "stream": stream, "layer": name, "shape": [n, C, h, w], "count": count,
                             "ms": round(ms, 4), "bytes_mb": round(nbytes / 1e6, 2),
                             "gb_s": round(nbytes / ms / 1e6, 1), "hbm_fraction": round(nbytes / ms / 1e-3 / HBM, 3)})
    totals = {}
    for r in rows:
        k = "%s %s" % (r["config"], r["stream"])
        totals[k] = round(totals.get(k, 0.0) + r["ms"] * r["count"], 3)
    return rows, totals


def _cfg(name, norm):
    cfg = getattr(UPSNetConfig, name)()
    for k in NORM_KEYS:
        setattr(cfg, k, norm)
    return cfg


def engine(iters):
    out = {}
    for name, (H, W) in (("cityscapes_r50", (1024, 2048)), ("coco_r50", (800, 1344))):
        inp = synthetic_input(H, W, seed=1, device=DEV)
        for norm in ("none", "group_norm"):
            m = synthetic_model(_cfg(name, norm), seed=0, device=DEV)
            for prec in ("bf16x3", "bf16"):
                U.set_precision(prec)
                with torch.no_grad():
                    m._run_static(inp["data"], inp["im_info"][0])
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(iters):
                        m._run_static(inp["data"], inp["im_info"][0])
                    torch.cuda.synchronize()
                out["%s %s %s" % (name, norm, prec)] = round(iters / (time.perf_counter() - t0), 2)
            del m
            torch.cuda.empty_cache()
    U.set_precision("fp32")
    return out


def train_step(iters):
    import train_forward_oracle as TF
    from upsnet_b200.training import PanopticLabels, RPNTargets
    H, W = 512, 1024
    out = {}
    for norm in ("none", "group_norm"):
        m = synthetic_model(_cfg("cityscapes_r50", norm), seed=0, device=DEV)
        entry, lmap = TF.synthetic_entry(1, H, W, 8)
        label = {"roidb": entry}
        np.random.seed(0)
        label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, DEV))
        label.update(PanopticLabels(dataset="cityscapes").from_roidb(entry, lmap, (H, W), 1.0, DEV))
        data = {"data": TF.image(2, H, W).to(DEV), "im_info": np.array([[H, W, 1.0]], np.float32)}
        U.set_precision("bf16x3")

        def step():
            m.zero_grad(set_to_none=True)
            np.random.seed(5)
            o = m(data, label)
            sum(o[k] for k in TF.LOSSES).backward()
        step()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
        out["cityscapes_r50 512x1024 %s step_ms" % norm] = round((time.perf_counter() - t0) / iters * 1e3, 2)
        del m
        torch.cuda.empty_cache()
    U.set_precision("fp32")
    return out


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    res = {"card": card()}
    rows, totals = pass_table(iters)
    res["passes"], res["gn_ms_per_image"] = rows, totals
    res["engine_images_s"] = engine(iters)
    res["train_step"] = train_step(max(3, iters // 10))
    res["card_after"] = card()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
