"""Plain, differentiable torch restatement of the training operators, evaluated in float64 (or any float dtype) on the CPU or
the device, and the error bounds the GPU backward tests measure against.

* deform_conv: DCN v1 / v2 forward (operators/src/deform_conv_kernel.cu, mod_deform_conv_kernel.cu): per tap the sample
  sits at ho*sh - ph + ki*dh + dh_off (same for w), counts only for -1 < h < H and -1 < w < W, and is a bilinear blend of
  its floor corners, each corner only if it lies inside the image; times the mask (v2), then the GEMM with the weight and
  the bias.  Autograd of it gives d(x), d(offset), d(mask), d(weight), d(bias).
  The sample positions are rounded the way the kernels compute them: integer base + fp32 offset in fp32.  Everything after
  that is in the working dtype.  Without the rounding, a sample within fp32 rounding of an integer could floor differently
  in the two computations.
* roi_align: Caffe2 ROIAlign (aligned=False) of roi_align_kernel.cu: extent max(size, 1), sr x sr grid (adaptive
  ceil(size / pooled) when sr <= 0), samples with y < -1 or y > H skipped, clamped to the last row / column.  The blend
  is separable, so each roi is A_y @ feat @ A_x^T with sparse per-axis weight matrices.
* fpn_levels: floor(2 + log2(sqrt(w*h)/224 + 1e-6)) clipped to [0, 3] with w = x2 - x1 + 1, in float32 like numpy.

The *_bounds functions give, per output element, the sum of the absolute values of the terms that make it up (fp64).
A kernel that computes the same sums in fp32 is within a small multiple of fp32 epsilon of that bound; see `check`.
The keyword arguments `right_guard` and `shift` build deliberately wrong variants for the sensitivity test.
"""
import math

import numpy as np
import torch

# Largest observed |kernel - fp64| / bound on an H100 is a few times below these (tests/test_gpu_backward.py prints it).
TOL = {"dcn_y": 8e-7, "dcn_dx": 8e-7, "dcn_doffset": 8e-7, "dcn_dmask": 6e-7, "dcn_dweight": 8e-7, "dcn_dbias": 2e-7,
       "roi_y": 2e-6, "roi_dfeat": 2e-6}
ATOL = 1e-6


def check(got, want, bound, c, atol=ATOL, slack=None):
    """(ok, worst (err - slack) / bound): element-wise |got - want| <= c * bound + slack + atol.  `slack` is the part of
    the error that does not scale with epsilon times the terms (ROIAlign: the rounding of the sample positions)."""
    err = (got.detach().double() - want.detach().double()).abs()
    bound = bound.detach().double().to(err.device)
    if slack is not None:
        err = err - slack.detach().double().to(err.device)
    ok = bool((err <= c * bound + atol).all())
    ratio = float((err / bound.clamp_min(1e-30)).masked_fill(err <= 0, 0).max()) if err.numel() else 0.0
    return ok, ratio


# ------------------------------------------------------------------------------------------------
# deformable convolution v1 / v2
# ------------------------------------------------------------------------------------------------
def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _corners(x, offset, kh, kw, stride, padding, dilation, offset32=None, right_guard=0, shift=0.0, fp32_positions=True):
    """The four bilinear corners of every sample: list of (value [N,C,K,Ho,Wo], weight [N,K,Ho,Wo] (0 where the corner is
    not used), used [N,K,Ho,Wo]), and the fractional positions lh, lw."""
    N, C, H, W = x.shape
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    K, Ho, Wo = kh * kw, offset.shape[2], offset.shape[3]
    dev = x.device
    tap = torch.arange(K, device=dev)
    base_h = (torch.arange(Ho, device=dev)[None, :, None] * sh - ph + (tap // kw)[:, None, None] * dh)      # [K,Ho,1]
    base_w = (torch.arange(Wo, device=dev)[None, None, :] * sw - pw + (tap % kw)[:, None, None] * dw)       # [K,1,Wo]
    off = offset.view(N, K, 2, Ho, Wo)
    o32 = (offset if offset32 is None else offset32).detach().float().view(N, K, 2, Ho, Wo)

    def pos(base, o, o_32):
        p = base.to(x.dtype) + o.to(x.dtype)
        if not fp32_positions:
            return p + shift
        p_kernel = (base.float() + o_32).to(x.dtype) + shift          # fp32 arithmetic, as the kernels do
        return p + (p_kernel - p).detach()

    h, w = pos(base_h, off[:, :, 0], o32[:, :, 0]), pos(base_w, off[:, :, 1], o32[:, :, 1])
    inside = (h > -1) & (h < H) & (w > -1) & (w < W)
    hl, wl = h.detach().floor(), w.detach().floor()
    lh, lw = h - hl, w - wl
    hl, wl = hl.long(), wl.long()
    xf = x.reshape(N, C, H * W)
    out = []
    for ddy, ddx, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
        yy, xx = hl + ddy, wl + ddx
        ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1 - (right_guard if ddx else 0))
        idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).reshape(N, 1, -1).expand(N, C, -1)
        v = xf.gather(2, idx).view(N, C, K, Ho, Wo)
        out.append((v, wt * ok.to(x.dtype), ok.to(x.dtype)))
    return out, lh, lw


def deform_conv(x, offset, weight, bias=None, mask=None, stride=1, padding=0, dilation=1, offset32=None, right_guard=0,
                shift=0.0, fp32_positions=True):
    """y [N,Cout,Ho,Wo] of DCN v1 (mask None) or v2 (mask [N,K,Ho,Wo], already activated).  offset32: the fp32 offsets
    whose rounding the sample positions take (default: `offset` itself); fp32_positions=False keeps them in the working
    dtype (for finite differences)."""
    N, C = x.shape[:2]
    Cout, _, kh, kw = weight.shape
    K, Ho, Wo = kh * kw, offset.shape[2], offset.shape[3]
    corners, _, _ = _corners(x, offset, kh, kw, stride, padding, dilation, offset32, right_guard, shift, fp32_positions)
    col = sum(v * wt[:, None] for v, wt, _ in corners)
    if mask is not None:
        col = col * mask.view(N, 1, K, Ho, Wo)
    y = torch.einsum("ok,nkp->nop", weight.reshape(Cout, C * K), col.reshape(N, C * K, Ho * Wo)).view(N, Cout, Ho, Wo)
    return y if bias is None else y + bias.view(1, Cout, 1, 1)


def deform_conv_bounds(x, offset, weight, bias, mask, dy, stride=1, padding=0, dilation=1):
    """Sums of absolute terms (fp64) of y and of every gradient for the output gradient dy."""
    x, offset, weight, dy = (t.detach().double() for t in (x, offset, weight, dy))
    N, C = x.shape[:2]
    Cout, _, kh, kw = weight.shape
    K, Ho, Wo = kh * kw, offset.shape[2], offset.shape[3]
    corners, lh, lw = _corners(x.abs(), offset, kh, kw, stride, padding, dilation)
    am = torch.ones(N, K, Ho, Wo, dtype=torch.float64, device=x.device) if mask is None else mask.detach().double().abs()
    col_nm = sum(v * wt[:, None] for v, wt, _ in corners).detach()          # bilinear of |x|
    col = col_nm * am[:, None]
    wa = weight.abs().reshape(Cout, C * K)
    dya = dy.abs().reshape(N, Cout, Ho * Wo)
    b = {"y": torch.einsum("ok,nkp->nop", wa, col.reshape(N, C * K, -1)).view(N, Cout, Ho, Wo)}
    if bias is not None:
        b["y"] = b["y"] + bias.detach().double().abs().view(1, Cout, 1, 1)
        b["bias"] = dya.sum((0, 2))
    b["weight"] = torch.einsum("nop,nkp->ok", dya, col.reshape(N, C * K, -1)).view_as(weight)
    dcol = torch.einsum("ok,nop->nkp", wa, dya).view(N, C, K, Ho, Wo)
    b["mask"] = (dcol * col_nm).sum(1)
    gh, gw = lh.detach(), lw.detach()
    coef_h = [1 - gw, gw, 1 - gw, gw]          # |d weight / dh| of the four corners
    coef_w = [1 - gh, 1 - gh, gh, gh]
    b_h = sum((dcol * v).sum(1) * ok * ch for (v, _, ok), ch in zip(corners, coef_h)) * am
    b_w = sum((dcol * v).sum(1) * ok * cw for (v, _, ok), cw in zip(corners, coef_w)) * am
    b["offset"] = torch.stack((b_h, b_w), 2).view(N, 2 * K, Ho, Wo)
    x0 = torch.zeros_like(x, requires_grad=True)
    with torch.enable_grad():
        y0 = deform_conv(x0, offset, weight.abs(), None, am, stride, padding, dilation)
        (b["x"],) = torch.autograd.grad(y0, x0, dy.abs())
    return b


# ------------------------------------------------------------------------------------------------
# ROIAlign (Caffe2, aligned=False) and the FPN level rule
# ------------------------------------------------------------------------------------------------
def _axis_weights(start, size, n_bins, grid, extent, dtype, dev, shift, f):
    """[n_bins, extent] weights of one axis (sum over the grid samples of each bin), and the same with each used tap
    weighted 1 (for the position-rounding term of the bound).  Positions in the numpy float type f (float32 like the
    kernel)."""
    bin_sz = f(size / f(n_bins))
    i = np.arange(n_bins, dtype=f).repeat(grid)
    s = np.tile(np.arange(grid, dtype=f), n_bins)
    pos = (f(start) + i * bin_sz + (s + f(0.5)) * bin_sz / f(grid)).astype(f)
    y = torch.from_numpy(pos.astype(np.float64) + shift).to(dev)
    valid = ~((y < -1) | (y > extent))
    y = y.clamp(min=0)
    lo = y.floor().long()
    top = lo >= extent - 1
    lo = torch.where(top, extent - 1, lo)
    hi = torch.where(top, extent - 1, lo + 1)
    y = torch.where(top, lo.double(), y)
    ly = (y - lo).to(dtype)
    bins = torch.arange(n_bins, device=dev).repeat_interleave(grid)
    A = torch.zeros(n_bins, extent, dtype=dtype, device=dev)
    T = torch.zeros(n_bins, extent, dtype=torch.float64, device=dev)
    v = valid.to(dtype)
    A.index_put_((bins, lo), (1 - ly) * v, accumulate=True)
    A.index_put_((bins, hi), ly * v, accumulate=True)
    T.index_put_((bins, lo), valid.double(), accumulate=True)
    T.index_put_((bins, hi), valid.double(), accumulate=True)
    return A, T


def _roi_geometry(roi, PH, PW, scale, sr, f):
    sc = f(scale)
    x1, y1, x2, y2 = (f(v) * sc for v in roi[1:5])
    rw, rh = max(f(x2 - x1), f(1)), max(f(y2 - y1), f(1))
    gh = sr if sr > 0 else int(math.ceil(f(rh / f(PH))))
    gw = sr if sr > 0 else int(math.ceil(f(rw / f(PW))))
    return int(round(float(roi[0]))), y1, rh, gh, x1, rw, gw


def _roi_one(feat, roi, PH, PW, scale, sr, shift, f=np.float32):
    b, y1, rh, gh, x1, rw, gw = _roi_geometry(roi, PH, PW, scale, sr, f)
    H, W = feat.shape[2:]
    Ay, Ty = _axis_weights(y1, rh, PH, gh, H, feat.dtype, feat.device, shift, f)
    Ax, Tx = _axis_weights(x1, rw, PW, gw, W, feat.dtype, feat.device, shift, f)
    # position rounding: the kernel and this restatement round each position within a few ulps of |start| + extent
    slack_y, slack_x = 2.0 ** -20 * (abs(float(y1)) + float(rh) + 1), 2.0 ** -20 * (abs(float(x1)) + float(rw) + 1)
    return b, Ay, Ax, Ty * slack_y, Tx * slack_x, gh * gw


def roi_align(feat, rois, PH, PW, scale, sr=2, shift=0.0, fp32_positions=True):
    """[R,C,PH,PW] from feat [B,C,H,W] (any float dtype, differentiable) and rois [R,5] (batch, x1, y1, x2, y2).
    fp32_positions=False computes the sample positions in float64 (as torchvision does for float64 input)."""
    R, C = rois.shape[0], feat.shape[1]
    f = np.float32 if fp32_positions else np.float64
    outs = []
    for roi in rois.detach().to(torch.float32 if fp32_positions else torch.float64).cpu().numpy():
        b, Ay, Ax, _, _, cnt = _roi_one(feat, roi, PH, PW, scale, sr, shift, f)
        outs.append(torch.einsum("ph,chw,qw->cpq", Ay, feat[b], Ax) / cnt)
    return torch.stack(outs) if outs else feat.new_zeros(R, C, PH, PW) + 0 * feat.sum()


def roi_align_bounds(feat, rois, PH, PW, scale, sr, dout):
    """Sums of absolute terms of y and of d(feat) for the output gradient dout ("y", "feat"), and the error the rounding of
    the sample positions can add on top ("y_slack", "feat_slack"): a position off by d moves two tap weights by d."""
    fa = feat.detach().double().abs()
    da = dout.detach().double().abs()
    by, sy, bf, sf = [], [], torch.zeros_like(fa), torch.zeros_like(fa)
    for n, roi in enumerate(rois.detach().float().cpu().numpy()):
        b, Ay, Ax, Sy, Sx, cnt = _roi_one(fa, roi, PH, PW, scale, sr, 0.0)
        Ay, Ax = Ay.double(), Ax.double()
        by.append(torch.einsum("ph,chw,qw->cpq", Ay, fa[b], Ax) / cnt)
        sy.append((torch.einsum("ph,chw,qw->cpq", Sy, fa[b], Ax) + torch.einsum("ph,chw,qw->cpq", Ay, fa[b], Sx)) / cnt)
        bf[b] += torch.einsum("ph,cpq,qw->chw", Ay, da[n], Ax) / cnt
        sf[b] += (torch.einsum("ph,cpq,qw->chw", Sy, da[n], Ax) + torch.einsum("ph,cpq,qw->chw", Ay, da[n], Sx)) / cnt
    shape = (rois.shape[0], fa.shape[1], PH, PW)
    return {"y": torch.stack(by) if by else fa.new_zeros(shape), "y_slack": torch.stack(sy) if sy else fa.new_zeros(shape),
            "feat": bf, "feat_slack": sf}


def fpn_levels(rois):
    """Index into [P2..P5] of every roi (fpn_roi_align.py's rule in float32)."""
    r = rois.detach().float().cpu().numpy()
    w = r[:, 3] - r[:, 1] + np.float32(1)
    h = r[:, 4] - r[:, 2] + np.float32(1)
    with np.errstate(divide="ignore"):
        lv = np.floor(np.float32(2) + np.log2(np.sqrt(w * h) / np.float32(224) + np.float32(1e-6)))
    return np.clip(lv, 0, 3).astype(np.int64)


def fpn_roi_align(feats, rois, PH, PW, scales, sr=2):
    """[R,C,PH,PW]: each roi pooled from the level fpn_levels picks."""
    lv = fpn_levels(rois)
    out = feats[0].new_zeros(rois.shape[0], feats[0].shape[1], PH, PW)
    for l in range(4):
        sel = np.nonzero(lv == l)[0]
        if len(sel):
            idx = torch.from_numpy(sel).to(out.device)
            out = out.index_copy(0, idx, roi_align(feats[l], rois[idx], PH, PW, scales[l], sr))
    return out


def fpn_roi_align_bounds(feats, rois, PH, PW, scales, sr, dout):
    lv = fpn_levels(rois)
    out = {k: torch.zeros(dout.shape, dtype=torch.float64, device=dout.device) for k in ("y", "y_slack")}
    out["feat"], out["feat_slack"] = [], []
    for l in range(4):
        sel = torch.from_numpy(np.nonzero(lv == l)[0]).to(dout.device)
        b = roi_align_bounds(feats[l], rois[sel], PH, PW, scales[l], sr, dout[sel])
        for k in ("y", "y_slack"):
            out[k][sel] = b[k]
        out["feat"].append(b["feat"])
        out["feat_slack"].append(b["feat_slack"])
    return out


def special_offsets(N, kh, kw, Ho, Wo, H, W, stride, padding, dilation, seed, frac=0.5, scale=1.5):
    """fp32 offsets [N, 2*kh*kw, Ho, Wo]: a share `frac` of the sample coordinates is placed exactly on the values where
    floor and the corner guards decide (integers, -1, H, (-1, 0), (H-1, H), beyond the image), the rest are random.  All
    values are dyadic, so the fp32 positions are exact."""
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    rng = np.random.default_rng(seed)
    K = kh * kw
    ki, kj = np.arange(K) // kw, np.arange(K) % kw
    base_h = (np.arange(Ho)[None, :, None] * sh - ph + ki[:, None, None] * dh) * np.ones((1, 1, Wo))
    base_w = (np.arange(Wo)[None, None, :] * sw - pw + kj[:, None, None] * dw) * np.ones((1, Ho, 1))

    def coord(base, E):
        sp = np.array([0, 1, E - 1, E - 2, -1, E, -0.5, -2.0 ** -10, -1 + 2.0 ** -10, E - 2.0 ** -10, E - 1.5, E - 0.5,
                       -1.5, -3, E + 2, E + 0.25, E // 2, E // 2 + 0.75])
        tgt = sp[rng.integers(0, len(sp), (N,) + base.shape)]
        rnd = base + np.round(rng.standard_normal((N,) + base.shape) * scale * 256) / 256
        return np.where(rng.uniform(size=(N,) + base.shape) < frac, tgt, rnd) - base

    off = np.stack([coord(base_h, H), coord(base_w, W)], 2).reshape(N, 2 * K, Ho, Wo)
    return torch.from_numpy(off.astype(np.float32))
