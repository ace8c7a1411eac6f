"""Plain-torch float64 oracle of the semantic head's ROI loss (train.fcn_with_roi_loss; models/fcn.py:102-106 and
models/resnet_upsnet.py:132-134), and the seeded cases of tests/golden/reference_fcn_roi_loss.npz.

* roi_align_weights: the reference's ROIAlign (aligned=False, roi extent >= 1, sampling_ratio x sampling_ratio samples,
  a sample outside [-1, H] x [-1, W] reads 0, clamps at 0 and H-1) as two separable interpolation matrices per roi,
  By [R,M,h] and Bx [R,M,w], so that RoIAlign(feat)[r,c,m,n] = sum By[r,m,y] feat[c,y,x] Bx[r,n,x].  The sample
  coordinates are computed in float32 as the kernels compute them (start + p*bin fused, then + (i+.5)*bin/sr); the
  weights in float64.
* loss_from_feat: the reference's composition, literally: the 512-channel concat of the four levels, RoIAlign, the 1x1
  score conv, cross-entropy with ignore_index 255 and reduce=False, then the mean over every cell.  It does not use
  the commutation of the score conv and ROIAlign.
* loss_from_score: the same loss from the score map (what FcnRoiLoss computes): RoIAlign of fcn_score plus
  bias * (1 - n_inside / count).  Differentiable in the score map and the bias; its per-element sums of |terms| give
  the a-priori error bounds of the device gradients.
"""
import hashlib

import torch
import torch.nn.functional as F

M, SR, SCALE = 28, 2, 0.25

# name: (seed, S, R, h, w, kind); h, w are the P2 (quarter-resolution) map size, multiples of 8
CASES = {
    "s19_r1": (11, 19, 1, 24, 32, "inside"),
    "s133_r90": (12, 133, 90, 16, 24, "random"),
    "partly_outside": (13, 19, 4, 16, 24, "outside"),
    "thin": (14, 19, 3, 16, 24, "thin"),
    "roi_all_ignored": (15, 19, 3, 16, 24, "ignored"),
}


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()[:16]


def boxes(g, R, h, w, kind):
    """[R,5] float32 rois (0, x1, y1, x2, y2) in image coordinates (4x the map)."""
    H4, W4 = 4.0 * h, 4.0 * w
    x1 = torch.rand(R, generator=g) * W4 * 0.7
    y1 = torch.rand(R, generator=g) * H4 * 0.7
    bw = 6.0 + torch.rand(R, generator=g) * W4 * 0.5
    bh = 6.0 + torch.rand(R, generator=g) * H4 * 0.5
    x2, y2 = x1 + bw, y1 + bh
    if kind == "inside":
        x1, y1, x2, y2 = x1 * 0.5 + 4, y1 * 0.5 + 4, torch.minimum(x2, torch.full_like(x2, W4 - 8)), \
            torch.minimum(y2, torch.full_like(y2, H4 - 8))
    elif kind == "outside":            # samples beyond -1 and beyond the far edge: the bias correction is not zero
        x1 = x1 - 0.6 * W4
        y2 = y2 + 0.8 * H4
    elif kind == "thin":               # under one map pixel wide / high: the extent is forced to 1
        x2 = x1 + 2.5
        y2[1:] = y1[1:] + 1.0
    return torch.cat([torch.zeros(R, 1), torch.stack([x1, y1, x2, y2], 1)], 1).float()


def case(name):
    """The seeded inputs of a case: the four subnet outputs (P2..P5 resolution, 128 channels each), the score conv,
    the rois and seg_roi_gt (int64, 255 mixed in)."""
    seed, S, R, h, w, kind = CASES[name]
    g = torch.Generator().manual_seed(seed)
    levels = [torch.randn(1, 128, h >> l, w >> l, generator=g) for l in range(4)]
    weight = torch.randn(S, 512, 1, 1, generator=g) * 0.05
    bias = torch.randn(S, generator=g) * 0.5
    rois = boxes(g, R, h, w, kind)
    seg = torch.randint(0, S, (R, M, M), generator=g)
    seg[torch.rand(R, M, M, generator=g) < 0.2] = 255
    if kind == "ignored":
        seg[1] = 255
    return {"levels": levels, "weight": weight, "bias": bias, "rois": rois, "seg": seg}


def inputs_digest(c):
    return "".join(digest(t) for t in c["levels"] + [c["weight"], c["bias"], c["rois"], c["seg"]])


def _coords(start, binsz, K, sr):
    k = torch.arange(K, device=start.device)
    p, i = (k // sr), (k % sr)
    a = (p.double()[None] * binsz.double()[:, None] + start.double()[:, None]).float()   # fused multiply-add
    return a + (((i.float() + 0.5)[None] * binsz[:, None]).double() / sr).float()


def _axis(coord, n, sr):
    """[R,K] float32 sample coordinates on an axis of n pixels -> [R,M,n] float64 weights (mean over the sr samples
    of each bin) and [R,M] float64 share of the samples inside."""
    R, K = coord.shape
    inside = ~((coord < -1.0) | (coord > float(n)))
    c = torch.clamp(coord, min=0.0)
    lo = torch.floor(c).long()
    top = lo >= n - 1
    lo = torch.where(top, torch.full_like(lo, n - 1), lo)
    hi = torch.where(top, lo, lo + 1)
    c = torch.where(top, lo.float(), c)
    l = c.double() - lo.double()
    wts = torch.zeros(R, K, n, dtype=torch.float64, device=coord.device)
    wts.scatter_add_(2, lo[..., None], ((1.0 - l) * inside)[..., None])
    wts.scatter_add_(2, hi[..., None], (l * inside)[..., None])
    return wts.view(R, K // sr, sr, n).sum(2) / sr, inside.double().view(R, K // sr, sr).sum(2) / sr


def roi_align_weights(rois, h, w, mask_size=M, scale=SCALE, sr=SR):
    """(By [R,M,h], Bx [R,M,w], inside [R,M,M]): the separable ROIAlign weights and each cell's n_inside / count."""
    r = rois.float()
    sc = torch.tensor(scale, dtype=torch.float32, device=r.device)
    rsw, rsh, rew, reh = r[:, 1] * sc, r[:, 2] * sc, r[:, 3] * sc, r[:, 4] * sc
    # float32 quotients rounded once, as the kernels' division (torch may divide by a scalar through its reciprocal)
    bsw = (torch.clamp(rew - rsw, min=1.0).double() / mask_size).float()
    bsh = (torch.clamp(reh - rsh, min=1.0).double() / mask_size).float()
    K = mask_size * sr
    By, iy = _axis(_coords(rsh, bsh, K, sr), h, sr)
    Bx, ix = _axis(_coords(rsw, bsw, K, sr), w, sr)
    return By, Bx, iy[:, :, None] * ix[:, None, :]


def feat_of(levels):
    p2, p3, p4, p5 = [t.double() for t in levels]
    up = lambda t, f: F.interpolate(t, None, f, mode="bilinear", align_corners=False)  # noqa: E731
    return torch.cat([p2, up(p3, 2), up(p4, 4), up(p5, 8)], 1)


def ce_mean(score, seg):
    return F.cross_entropy(score, seg, ignore_index=255, reduction="none").mean()


def loss_from_feat(levels, weight, bias, rois, seg, scale=SCALE):
    """The reference's composition in float64: RoIAlign of the 512-channel concat, then the score conv, then the loss."""
    feat = feat_of(levels)[0]
    By, Bx, _ = roi_align_weights(rois, feat.shape[1], feat.shape[2], seg.shape[1], scale)
    rf = torch.einsum("rmy,cyx,rnx->rcmn", By, feat, Bx)
    score = torch.einsum("rcmn,sc->rsmn", rf, weight.double().flatten(1)) + bias.double()[None, :, None, None]
    return ce_mean(score, seg)


def roi_scores(fcn, bias, rois, mask_size=M, scale=SCALE, correct_bias=True):
    """[R,S,M,M] float64 roi scores sampled from the score map fcn [S,h,w] (+ the bias share ROIAlign's zeros remove)."""
    By, Bx, inside = roi_align_weights(rois, fcn.shape[1], fcn.shape[2], mask_size, scale)
    s = torch.einsum("rmy,syx,rnx->rsmn", By, fcn.double(), Bx)
    if correct_bias:
        s = s + bias.double()[None, :, None, None] * (1.0 - inside)[:, None]
    return s


def loss_from_score(fcn, bias, rois, seg, mask_size=M, scale=SCALE, correct_bias=True, mean_over_valid=False):
    """FcnRoiLoss in float64 from fcn [S,h,w]; the two switches plant the faults the tests must reject."""
    score = roi_scores(fcn, bias, rois, mask_size, scale, correct_bias)
    valid = (seg >= 0) & (seg < score.shape[1])
    t = torch.where(valid, seg, torch.zeros_like(seg))
    lse = torch.logsumexp(score, 1)
    cell = (lse - score.gather(1, t[:, None])[:, 0]) * valid
    return cell.sum() / (valid.sum() if mean_over_valid else seg.numel())


def grad_bounds(fcn, bias, rois, seg, mask_size=M, scale=SCALE, grad_out=1.0):
    """Per-element sums of |terms| of d fcn_score [S,h,w] and d bias [S]: every cell contributes tap weight *
    (softmax + onehot) * |grad_out| / (R*M*M), the two parts of its gradient counted apart."""
    score = roi_scores(fcn, bias, rois, mask_size, scale)
    valid = (seg >= 0) & (seg < score.shape[1])
    p = torch.softmax(score, 1) * valid[:, None]
    onehot = F.one_hot(torch.where(valid, seg, torch.zeros_like(seg)), score.shape[1]).permute(0, 3, 1, 2) * valid[:, None]
    a = (p + onehot) * abs(grad_out) / seg.numel()
    By, Bx, inside = roi_align_weights(rois, fcn.shape[1], fcn.shape[2], mask_size, scale)
    return torch.einsum("rmy,rsmn,rnx->syx", By, a, Bx), (a * (1.0 - inside)[:, None]).sum((0, 2, 3))
