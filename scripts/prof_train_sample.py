"""Device time of one training sample (TrainingSample.sample) per phase: python scripts/prof_train_sample.py [calls]

Cases: Cityscapes 1024x2048 (30 instances) at scales 800 and 1024, flipped and not, and COCO 600x1000 at scale 800
(an 800x1333 blob, 15 instances, one crowd), from synthetic images, label maps and entries built from a seed.
Phases, each timed on its own over `calls` repetitions:
  h2d_image_ms / h2d_label_ms  the uint8 image and label map from pinned host memory (CUDA events)
  prep_ms                      ops.prep_image: mean, flip, bilinear resize, pad, HWC -> CHW (CUDA events)
  rpn_targets_ms               RPNTargets.from_roidb as issued from Python: host box scaling, its upload, the launch
  label_maps_ms                PanopticLabels.launch on prepared tables: seg_gt, seg_gt_4x, mask_gt, seg_roi_gt
  roidb_packing_host_ms        host time of PanopticLabels.pack_roidb + prepare (polygons, index tables, their upload)
  sample_wall_ms               one whole sample() from pinned host arrays, host clock around a device synchronise
with the card and its power limit read in the same run."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import label_oracle as LO  # noqa: E402
import train_sample_cases as TS  # noqa: E402
from prof_rpn_targets import card, events_ms  # noqa: E402
from upsnet_b200 import prep_image  # noqa: E402
from upsnet_b200.training import TrainingSample  # noqa: E402

# (name, dataset, h, w, G, target size, flipped)
CASES = [("cityscapes_800", "cityscapes", 1024, 2048, 30, 800, False),
         ("cityscapes_800_flip", "cityscapes", 1024, 2048, 30, 800, True),
         ("cityscapes_1024", "cityscapes", 1024, 2048, 30, 1024, False),
         ("cityscapes_1024_flip", "cityscapes", 1024, 2048, 30, 1024, True),
         ("coco_800x1333_flip", "coco", 600, 1000, 15, 800, True)]


def host_ms(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def measure(case, n):
    name, dataset, h, w, G, target, flipped = case
    dev = torch.device("cuda", 0)
    base = LO.random_entry(np.random.default_rng(7), h, w, G, dataset)
    entry = TS.flip_entry(base) if flipped else base
    image = torch.from_numpy(TS.image_bgr(h, w, 7)).pin_memory()
    label_map = torch.from_numpy(LO.label_png(h, w, 7)).pin_memory()
    cfg = TS.CONFIGS[dataset]
    ts = TrainingSample(dataset=dataset, scales=(target,), max_size=cfg["max_size"], with_roi=cfg["with_roi"])
    _, s = ts.draw_scale(h, w)
    ho, wo = int(np.rint(h * s)), int(np.rint(w * s))
    imd, labd = image.to(dev), label_map.to(dev)

    def pack(i=0):
        pk = ts.labels.pack_roidb(entry, s, dev)
        return pk, ts.labels.prepare((h, w), pk, (ho, wo), s, flipped, dev)

    pk, tab = pack()
    phases = {
        "h2d_image_ms": lambda i: imd.copy_(image, non_blocking=True),
        "h2d_label_ms": lambda i: labd.copy_(label_map, non_blocking=True),
        "prep_ms": lambda i: prep_image(imd, ts.pixel_means, s, ts.stride, flip=flipped),
        "rpn_targets_ms": lambda i: ts.rpn.from_roidb(entry, s, dev, seed=i),
        "label_maps_ms": lambda i: ts.labels.launch(labd, pk, tab, mask_dtype=torch.int64),
    }
    res = {"case": name, "blob": None, "scale": s, "calls": n}
    for k, fn in phases.items():
        fn(0)
        torch.cuda.synchronize()
        res[k] = round(events_ms(fn, n), 4)
    res["roidb_packing_host_ms"] = round(host_ms(pack, n), 4)
    data, label = ts.sample(entry, image, label_map, dev, seed=0)
    res["blob"] = list(data["data"].shape)
    res["sample_wall_ms"] = round(host_ms(lambda i: ts.sample(entry, image, label_map, dev, seed=i), n), 4)
    res["phase_sum_ms"] = round(sum(res[k] for k in phases) + res["roidb_packing_host_ms"], 4)
    return res


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"card": card(), "cases": [measure(c, n) for c in CASES], "card_after": card()}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
