"""Generates tests/golden/reference_kernels.npz: outputs of the reference's own CUDA kernels (ROIAlign, NMS, deformable
conv; oracle/_ref/libupsnet_ref.so, built by __graft_entry__.build() where the reference checkout is present) on the
inputs of the comparisons in tests/test_gpu_parity.py.  Needs a GPU and oracle/_ref.
Run: python tests/golden/make_reference_kernels.py

Large outputs are stored as a fixed sample (seed 1234, SAMPLE flat elements, sorted indices `<key>_idx`) so that the
file stays small; the tests compare the same elements."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import oracle as O  # noqa: E402
from test_gpu_parity import DCN_CFGS, rand_rois  # noqa: E402

SAMPLE = 4096


def sample(out, key, a):
    a = np.asarray(a, np.float32).reshape(-1)
    if a.size <= SAMPLE:
        out[key] = a
        return
    idx = np.sort(np.random.default_rng(1234).choice(a.size, SAMPLE, replace=False)).astype(np.int64)
    out[key + "_idx"] = idx
    out[key] = a[idx]


def main():
    dev = torch.device("cuda", 0)
    ref = O.RefKernels()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = {}
    g = np.load(os.path.join(HERE, "oracle_ops.npz"))
    sample(out, "ra_golden", ref.roi_align(t(g["ra_feat"]), t(g["ra_rois"]), 7, 7, 0.25).cpu().numpy())
    for ph in (7, 14):          # test_roi_align_config1_nchw_and_nhwc
        torch.manual_seed(0)
        rng = np.random.default_rng(0)
        feat = torch.randn(1, 256, 256, 256)
        rois = rand_rois(rng, 32, 1, 1024, 16, 512)
        sample(out, "ra_config1_%d" % ph, ref.roi_align(feat.to(dev), t(rois), ph, ph, 0.25).cpu().numpy())
    gr = np.load(os.path.join(HERE, "reference_numpy.npz"))
    for i in range(int(gr["nms_cases"])):
        out["nms_golden%d" % i] = np.asarray(ref.nms(gr["nms%d_dets" % i], float(gr["nms%d_thresh" % i])), np.int64)
    rng = np.random.default_rng(11)      # test_nms_dense_random_bit_exact: same draws in the same order
    for n, extent in [(1, 50), (64, 80), (65, 80), (129, 100), (1000, 250), (4097, 600), (8000, 1200)]:
        c = rng.uniform(0, extent, (n, 2)); s = np.exp(rng.uniform(np.log(16), np.log(128), (n, 2)))
        scores = (rng.permutation(n) + 1.0) / (n + 1)
        d = np.concatenate([c - s / 2, c + s / 2, scores[:, None]], 1).astype(np.float32)
        if n <= 4097:
            out["nms_dense%d" % n] = np.asarray(ref.nms(d, 0.5), np.int64)
    sample(out, "dcn_golden", ref.deform_conv(t(g["dcn_x"]), t(g["dcn_off"]), t(g["dcn_w"]), t(g["dcn_b"]), pad=1, dg=2).cpu().numpy())
    for ci, cfg in enumerate(DCN_CFGS):  # test_dcn_vs_oracle
        for modulated in (False, True):
            rng = np.random.default_rng(21)
            N, Cin, Cout, H, W = cfg["N"], cfg["Cin"], cfg["Cout"], cfg["H"], cfg["W"]
            Ho = O.conv_out(H, cfg["pad"], cfg["dil"], 3, cfg["stride"]); Wo = O.conv_out(W, cfg["pad"], cfg["dil"], 3, cfg["stride"])
            x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
            w = (rng.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cin * 9)).astype(np.float32)
            b = rng.standard_normal(Cout).astype(np.float32)
            off = (rng.standard_normal((N, 18 * cfg["dg"], Ho, Wo)) * 2.5).astype(np.float32)
            mask = (rng.uniform(0, 2, (N, 9 * cfg["dg"], Ho, Wo))).astype(np.float32) if modulated else None
            r = ref.deform_conv(t(x), t(off), t(w), t(b), None if mask is None else t(mask), cfg["stride"], cfg["pad"],
                                cfg["dil"], cfg["dg"])
            sample(out, "dcn_cfg%d_%d" % (ci, int(modulated)), r.cpu().numpy())
    np.savez_compressed(os.path.join(HERE, "reference_kernels.npz"), **out)
    print("wrote reference_kernels.npz:", len(out), "arrays")


if __name__ == "__main__":
    main()
