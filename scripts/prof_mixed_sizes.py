"""Throughput of a COCO-like mix of image sizes through the inference engine:
python scripts/prof_mixed_sizes.py [n_images] [n_forward]

Model: the COCO R50 configuration with synthetic weights, at bf16x3 and at bf16.  Images: a seeded mix of original
sizes -- landscape, portrait, square, and elongated ones whose long side hits max_size -- as uint8 pinned host images,
resized and padded on the device by the reference's test-phase rule (target 800, max_size 1333).
Reported per precision:
  mixed_engine_images_s     the mixed-size PipelinedEngine (depth 4, lanes 2, masks), after one warm pass over every
                            padded shape, host clock around the whole stream ending in its last result
  forward_recapture_images_s  the first n_forward images through model.forward with the graph cache cleared before each
                            one: a warm-up and a capture per image, which is what a cache keyed on im_info costs on COCO,
                            where nearly every image has its own im_info
  fixed_engine_800x1344_images_s  a fixed-size PipelinedEngine, every image 800x1333 (padded 800x1344): the ceiling
  graphs_per_lane, padded_shapes, reserved_growth_per_later_capture_mb (what one more captured shape costs once each
  lane has its pool), max_memory_reserved_gb
with the card and its power limit read in the same run."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import upsnet_b200 as U  # noqa: E402
from prof_rpn_targets import card  # noqa: E402
from upsnet_b200.geometry import image_geometry  # noqa: E402
from upsnet_b200.model import UPSNetConfig  # noqa: E402
from upsnet_b200.synthetic import synthetic_model  # noqa: E402

TARGET, MAX_SIZE = 800, 1333
MEANS = (102.9801, 115.9465, 122.7717)


def size_mix(n, seed=0):
    """COCO-like original sizes: long side 640 (mostly) or 500, short side drawn per orientation; a few square and a few
    elongated images (aspect > 1333 / 800, so max_size binds)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        kind = rng.choice(["landscape", "portrait", "square", "elongated"], p=[0.55, 0.3, 0.08, 0.07])
        long_ = int(rng.choice([640, 640, 640, 500]))
        if kind == "square":
            out.append((long_, long_))
            continue
        short = int(rng.integers(260, 380)) if kind == "elongated" else int(rng.integers(330, 481))
        out.append((short, long_) if kind in ("landscape", "elongated") else (long_, short))
    return out


def images(sizes, seed=1):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).pin_memory() for h, w in sizes]


def stream(eng, imgs, depth):
    pending, t0 = [], time.perf_counter()
    for im in imgs:
        pending.append(eng.submit(im))
        if len(pending) >= depth:
            eng.result(pending.pop(0))
    for t in pending:
        eng.result(t)
    return len(imgs) / (time.perf_counter() - t0)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    n_fwd = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    dev = torch.device("cuda", 0)
    sizes = size_mix(n)
    imgs = images(sizes)
    geos = [image_geometry(h, w, TARGET, MAX_SIZE) for h, w in sizes]
    shapes = sorted({g.padded for g in geos})
    res = {"card": card(), "images": n, "padded_shapes": len(shapes), "sizes_head": sizes[:8]}
    for prec in ("bf16x3", "bf16"):
        U.set_precision(prec)
        m = synthetic_model(UPSNetConfig.coco_r50(), seed=0, device=dev)
        m.prepare()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        r = {}
        # mixed-size engine: one warm pass over every padded shape, then the timed stream
        depth = 4
        eng = U.PipelinedEngine(m, depth=depth, lanes=2, with_masks=True, target_size=TARGET, max_size=MAX_SIZE,
                                max_image_shape=(640, 640), pixel_means=MEANS)
        first = {}
        for g, im in zip(geos, imgs):
            first.setdefault(g.padded, im)
        reserved = [torch.cuda.memory_reserved()]
        for im in list(first.values()) * 2:             # twice: every shape on both lanes
            eng.result(eng.submit(im))
            torch.cuda.synchronize()
            reserved.append(torch.cuda.memory_reserved())
        steps = np.diff(reserved[2:])                    # growth per new (shape, lane) after the first capture of each lane
        r["graphs_per_lane"] = {str(lane): sum(1 for k in m._graphs if k[-1] == lane) for lane in (0, 1)}
        r["reserved_growth_per_later_capture_mb"] = {"median": float(np.median(steps) / 2 ** 20),
                                                     "max": float(np.max(steps) / 2 ** 20)}
        r["mixed_engine_images_s"] = stream(eng, imgs, depth)
        r["mixed_engine_images_s_repeat"] = stream(eng, imgs, depth)
        del eng
        # model.forward as it ran before: the graph cache was keyed on im_info too, so a new image meant a new capture
        fwd = []
        for im, g in zip(imgs[:n_fwd], geos[:n_fwd]):
            blob, _ = U.prep_image(im.to(dev), MEANS, g.scale)
            m._graphs = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m({"data": blob, "im_info": g.im_info[None]})
            torch.cuda.synchronize()
            fwd.append(time.perf_counter() - t0)
        r["forward_recapture_images_s"] = len(fwd) / sum(fwd)
        m._graphs = {}
        # ceiling: a fixed-size engine, every image 800x1344
        fixed_imgs = images([(800, 1333)] * 8, seed=2)
        eng = U.PipelinedEngine(m, np.array([[800, 1333, 1.0]], np.float32), depth=depth, lanes=2, with_masks=True,
                                pixel_means=MEANS)
        stream(eng, fixed_imgs, depth)
        r["fixed_engine_800x1344_images_s"] = stream(eng, fixed_imgs * (n // 8), depth)
        del eng
        torch.cuda.synchronize()
        r["max_memory_reserved_gb"] = torch.cuda.max_memory_reserved() / 2 ** 30
        res[prec] = r
        del m
        torch.cuda.empty_cache()
    U.set_precision("fp32")
    res["card_after"] = card()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
