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
* dcn_columns / dcn_gemm: the arithmetic of the inference DCN kernels per precision mode (bf16x3 on fp32 or pair
  activations, bf16), with planted faults; special_offsets(window=...) / window_origins: the window kernel's geometry.
"""
import math

import numpy as np
import torch

# Largest observed |kernel - fp64| / bound on an H100 is a few times below these (tests/test_gpu_backward.py prints it).
TOL = {"dcn_y": 8e-7, "dcn_dx": 8e-7, "dcn_doffset": 8e-7, "dcn_dmask": 6e-7, "dcn_dweight": 8e-7, "dcn_dbias": 2e-7,
       "roi_y": 2e-6, "roi_dfeat": 2e-6,
       # inference (tensor-core) DCN forward per precision mode: about 4x the worst ratio measured on an H100, far below
       # the a-priori 2.1e-4, 1.35e-4 and 3.5e-5 derived in tests/test_gpu_forward_fp64.py
       "dcn_x3_pair": 2e-5, "dcn_x3_f32": 1.2e-5, "dcn_bf16": 2.6e-6}
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
# the arithmetic of the inference (tensor-core) DCN kernels, restated for the reference of the bf16 path and for the
# sensitivity test of the forward tolerances
# ------------------------------------------------------------------------------------------------
def bf16_round(v, trunc=False):
    """v (float64) rounded to bf16 (8 significant bits), ties to even, or towards zero (trunc); float64 result."""
    m, e = torch.frexp(v)
    m = m * 256
    return torch.ldexp(torch.trunc(m) if trunc else torch.round(m), e - 8)


def half_ulp_bf16(v):
    """Half a bf16 ulp of |v| (0 where v == 0), float64."""
    _, e = torch.frexp(v.abs())
    return torch.where(v == 0, 0.0, torch.ldexp(torch.ones_like(v), e - 9))


def check_pair_split(store):
    """A pair tensor [..., 2C] is normalised: hi == bf16(hi + lo) and |lo| <= half an ulp of hi.  When o - hi lies just
    below half an ulp, lo = bf16(o - hi) rounds up to exactly half an ulp and hi + lo is a rounding midpoint (about 1 in
    1000 elements of Pair.from_float); there either neighbour is a nearest bf16 value, so hi passes if it is one of them."""
    c = store.shape[-1] // 2
    hi, lo = store[..., :c].double(), store[..., c:].double()
    v = hi + lo
    r = bf16_round(v)
    assert bool(((r == hi) | ((v - hi).abs() == (v - r).abs())).all()), "hi is not the bf16 rounding of hi + lo"
    assert bool((lo.abs() <= half_ulp_bf16(hi)).all()), "|lo| exceeds half an ulp of hi"


def split_bf16(v):
    """(hi, lo) = (bf16(v), bf16(v - hi)) of fp32 values v, as float64."""
    hi = bf16_round(v)
    return hi, bf16_round(v - hi)


def _fl32(v):
    return v.float().double()


def dcn_columns(x, offset, kh, kw, stride, padding, dilation, mask=None, mode="x3_f32", fault=None, window=None):
    """The blended samples [N, C, K, Ho, Wo] (float64 tensors holding the kernel's values) as the tensor-core gathers
    form them (csrc/igemm_tc.cu, csrc/dcn_win.cu).  Corner weights: the fp32 bilinear weight of each corner times the
    mask, in fp32, 0 for corners outside the image.
      'x3_f32'  fp32 activations x: fp32 FMA chain over the four corners, split into bf16 (hi, lo) -> (hi, lo)
      'x3_pair' pair activations x = (hi, lo): hi plane in an fp32 FMA chain, lo plane in a bf16 FMA chain
                (HMUL2 + 3 HFMA2) with bf16-rounded weights, the two added in fp32 and split -> (hi, lo)
      'bf16'    bf16 activations x: the weights rounded to bf16, then a bf16 FMA chain -> s
    Faults for the sensitivity test: 'right_guard', 'shift' (as in deform_conv), 'mask_hi_only' (x3: the lo plane of
    x, or of the split sample, without the mask), 'truncate' (bf16: the chain truncates instead of rounding),
    'window_edge' (window=(TW, TH): dcn_win.cu's in-window test one px too wide, reading the corner one past the window
    as 0)."""
    planes = x if mode == "x3_pair" else (x,)
    C = planes[0].shape[1]
    xs = torch.cat([p.float() for p in planes], 1)
    corners, _, _ = _corners(xs, offset, kh, kw, stride, padding, dilation, None, 1 if fault == "right_guard" else 0,
                             1 / 64 if fault == "shift" else 0.0)
    wts = [wt for _, wt, _ in corners]
    if fault == "window_edge":
        N, Ho, Wo = offset.shape[0], offset.shape[2], offset.shape[3]
        (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
        K = kh * kw
        base_h = (np.arange(Ho)[None, :, None] * sh - ph + (np.arange(K) // kw)[:, None, None] * dh) * np.ones((1, 1, Wo))
        base_w = (np.arange(Wo)[None, None, :] * sw - pw + (np.arange(K) % kw)[:, None, None] * dw) * np.ones((1, Ho, 1))
        o = offset.detach().float().double().cpu().numpy().reshape(N, K, 2, Ho, Wo)
        ox, oy, hl, wl, valid = window_origins(base_h + o[:, :, 0], base_w + o[:, :, 1], xs.shape[2], xs.shape[3], window)
        dx, dy = wl - ox, hl - oy
        inside = (dx >= 0) & (dx + 1 < WIN_W) & (dy >= 0) & (dy + 1 < WIN_H)
        wide = valid & ~inside & (dx >= 0) & (dx < WIN_W) & (dy >= 0) & (dy < WIN_H)      # the one-px-too-wide test
        drop_r = torch.from_numpy(wide & (dx + 1 == WIN_W)).to(xs.device)
        drop_b = torch.from_numpy(wide & (dy + 1 == WIN_H)).to(xs.device)
        wts = [wts[0], wts[1] * ~drop_r, wts[2] * ~drop_b, wts[3] * ~(drop_r | drop_b)]
    m32 = None if mask is None else mask.float()
    wm = [w if m32 is None else w * m32 for w in wts]                    # fp32, as the kernels' sample tables
    wm, wts = [w.double()[:, None] for w in wm], [w.double()[:, None] for w in wts]
    vals = [v.double() for v, _, _ in corners]
    if mode == "bf16":
        s = None
        for v, w in zip(vals, wm):
            s = bf16_round(bf16_round(w) * v + (0 if s is None else s), trunc=fault == "truncate")
        return s
    if mode == "x3_f32":
        w_hi = wts if fault == "mask_hi_only" else wm
        s = None
        for v, w in zip(vals, w_hi):
            s = _fl32(w * v + (0 if s is None else s))
        hi, lo = split_bf16(s)
        return (hi * mask.double()[:, None], lo) if fault == "mask_hi_only" and mask is not None else (hi, lo)
    assert mode == "x3_pair"
    acc, lacc = None, None
    for v, w, w_nm in zip(vals, wm, wts):
        acc = _fl32(w * v[:, :C] + (0 if acc is None else acc))
        lacc = bf16_round(bf16_round(w_nm if fault == "mask_hi_only" else w) * v[:, C:] + (0 if lacc is None else lacc))
    return split_bf16(_fl32(acc + lacc))


def dcn_gemm(col, weight, bias=None, mode="x3_f32", fault=None, dtype=torch.float32):
    """y [N, Cout, Ho, Wo] from the columns of dcn_columns: bf16 x bf16 products (exact) summed in `dtype`.
    x3: s_hi w_hi + s_lo w_hi + s_hi w_lo (fault 'drop_lohi': without s_lo w_hi); bf16: s w (weights bf16-exact)."""
    Cout = weight.shape[0]
    w2 = weight.double().reshape(Cout, -1)

    def mm(a, b):
        N, Ho, Wo = a.shape[0], a.shape[3], a.shape[4]
        return torch.einsum("ok,nkp->nop", b.to(dtype), a.reshape(N, -1, Ho * Wo).to(dtype)).view(N, Cout, Ho, Wo)
    if mode == "bf16":
        y = mm(col, w2)
    else:
        (s_hi, s_lo), (w_hi, w_lo) = col, split_bf16(w2)
        y = mm(s_hi, w_hi) + mm(s_hi, w_lo)
        if fault != "drop_lohi":
            y = y + mm(s_lo, w_hi)
    return y if bias is None else y + bias.to(dtype).view(1, Cout, 1, 1)


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


def hand_rois(H, W, scale, n_random, seed):
    """Hand-placed rois (image coordinates) on a [*, *, H, W] map at `scale`, then random ones on both images."""
    iw, ih = W / scale, H / scale
    hand = [[0, 4, 4, 60, 50], [1, 10, 20, 100, 90],              # plain, batch index 1
            [0, -20, -10, 30, 25], [1, iw - 30, ih - 40, iw + 30, ih + 10],   # partly outside
            [1, -100, -100, -60, -50], [0, iw + 8, 4, iw + 60, 40],           # entirely outside
            [0, iw - 1 / scale, 0, iw - 1 / scale, ih - 1 / scale],           # on the last column (zero width)
            [1, 0, ih - 1 / scale, iw - 1 / scale, ih - 1 / scale],           # on the last row
            [0, 0, 0, iw - 1 / scale, ih - 1 / scale],                         # the whole map
            [0, 10.25, 10.5, 10.75, 10.875], [1, 33.5, 7.25, 34.0, 7.5]]       # smaller than one pixel
    rng = np.random.default_rng(seed)
    cxy = rng.uniform(0, 1, (n_random, 2)) * np.array([iw, ih])
    sz = np.exp(rng.uniform(np.log(2), np.log(max(iw, ih)), (n_random, 2)))
    rnd = np.concatenate([rng.integers(0, 2, (n_random, 1)), cxy - sz / 2, cxy + sz / 2], 1)
    return torch.tensor(np.concatenate([np.array(hand, np.float64), rnd]), dtype=torch.float32)


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


def special_offsets(N, kh, kw, Ho, Wo, H, W, stride, padding, dilation, seed, frac=0.5, scale=1.5, window=None):
    """fp32 offsets [N, 2*kh*kw, Ho, Wo]: a share `frac` of the sample coordinates is placed exactly on the values where
    floor and the corner guards decide (integers, -1, H, (-1, 0), (H-1, H), beyond the image), the rest are random.  All
    values are dyadic, so the fp32 positions are exact.
    window=(TW, TH), stride 1 only: then the samples of every TW x TH tile of output pixels are rearranged for the window
    kernel (csrc/dcn_win.cu), see _place_window."""
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
        return np.where(rng.uniform(size=(N,) + base.shape) < frac, tgt, rnd)

    h, w = coord(base_h, H), coord(base_w, W)
    if window is not None:
        assert (sh, sw) == (1, 1), "the window kernel runs stride-1 layers only"
        _place_window(h, w, base_h, base_w, H, W, window, rng)
    off = np.stack([h - base_h, w - base_w], 2).reshape(N, 2 * K, Ho, Wo)
    return torch.from_numpy(off.astype(np.float32))


# ------------------------------------------------------------------------------------------------
# the window of csrc/dcn_win.cu: per tile of output pixels one WIN_W x WIN_H-pixel window of the input is staged in
# shared memory; samples with both corner columns and both corner rows inside it read it, the others (outliers) read
# global memory.
# ------------------------------------------------------------------------------------------------
WIN_W, WIN_H = 32, 20          # DW_WW, DW_WH


def _origin(hl, wl, cnt):
    """dcn_win.cu's window origin of one tile from the floors of its valid samples (int arrays) and their count: the
    corner bounding box if it fits, else centred on the mean floor (fp32 arithmetic, as the kernel)."""
    if cnt == 0:
        return 0, 0

    def axis(fl, size):
        lo, hi = int(fl.min()), int(fl.max()) + 1
        if hi - lo + 1 <= size:
            return lo
        return int(np.floor(np.float32(int(fl.sum())) / np.float32(cnt) + np.float32(1))) - size // 2
    return axis(wl, WIN_W), axis(hl, WIN_H)


def _tiles(N, Ho, Wo, tile):
    TW, TH = tile
    for n in range(N):
        for y0 in range(0, Ho, TH):
            for x0 in range(0, Wo, TW):
                yield n, slice(y0, min(y0 + TH, Ho)), slice(x0, min(x0 + TW, Wo))


def window_origins(h, w, H, W, tile):
    """Window origin (ox, oy) of every sample of h, w (float64 [N, K, Ho, Wo], exact fp32 sample coordinates) for the
    kernel's TW x TH tiles of output pixels, with the floors and the validity (-1 < h < H, -1 < w < W) of the samples."""
    valid = (h > -1) & (h < H) & (w > -1) & (w < W)
    hl, wl = np.floor(h).astype(np.int64), np.floor(w).astype(np.int64)
    ox, oy = np.zeros(h.shape, np.int64), np.zeros(h.shape, np.int64)
    for n, ys, xs in _tiles(h.shape[0], h.shape[2], h.shape[3], tile):
        v = valid[n, :, ys, xs]
        ox[n, :, ys, xs], oy[n, :, ys, xs] = _origin(hl[n, :, ys, xs][v], wl[n, :, ys, xs][v], int(v.sum()))
    return ox, oy, hl, wl, valid


def _place_window(h, w, base_h, base_w, H, W, tile, rng):
    """Rearrange the sample coordinates h, w ([N, K, Ho, Wo], in place) tile by tile, cycling through three modes:
    0 / 1  every sample inside the image, the corner bounding box exactly WIN_W - 1, WIN_W or WIN_W + 1 px wide (mode 0)
           or WIN_H - 1, WIN_H, WIN_H + 1 px tall (mode 1): both sides of the kernel's `box fits -> window at the box`
           test, and with a fitting box, samples whose high corner is the window's last column / row.
    2      one far outlier (at the far image corner) makes the box too large, so the window is centred on the mean
           sample; then samples are placed on the window's last column and row -- integer ones, whose zero-weight high
           corner lies one past the window, and fractional ones, which leave it -- one px before them, and one px before
           the window's first column and row: both sides of the per-sample `both corners inside -> window, else
           global-memory outlier` test."""
    N, K, Ho, Wo = h.shape
    for t, (n, ys, xs) in enumerate(_tiles(N, Ho, Wo, tile)):
        th, tw = h[n, :, ys, xs], w[n, :, ys, xs]                # views
        bh, bw = base_h[:, ys, xs], base_w[:, ys, xs]
        mode, d = t % 3, (t // 3) % 3 - 1
        # the bulk: inside the tile's own base footprint and inside the image (all valid, the box fits)
        np.clip(th, max(bh.min(), 0), min(bh.max(), H - 1), out=th)
        np.clip(tw, max(bw.min(), 0), min(bw.max(), W - 1), out=tw)
        if mode < 2:
            a, E, size = (tw, W, WIN_W) if mode == 0 else (th, H, WIN_H)
            span = size + d                                      # corner box = max floor + 1 - min floor + 1
            lo = min(max(a.min(), 0), E - span)
            if lo < 0:
                continue                                         # the image is narrower than the span
            top = lo + span - 2 + (0.5 if t % 2 else 0.0)        # the largest floor is lo + span - 2
            np.clip(a, lo, top, out=a)
            a.flat[0], a.flat[-1] = lo, top
            continue
        far = (0 if xs.start > W / 2 else W - 1, 0 if ys.start > H / 2 else H - 1)
        tw.flat[K // 2 * tw.shape[1] * tw.shape[2]], th.flat[K // 2 * th.shape[1] * th.shape[2]] = far
        slots = rng.choice(np.arange(1, th.size), size=8, replace=False)
        for _ in range(4):                                       # the placed samples move the mean a little
            ox, oy = _origin(np.floor(th).astype(np.int64).ravel(), np.floor(tw).astype(np.int64).ravel(), th.size)
            xm, ym = ox + WIN_W // 2, oy + WIN_H // 2
            # (row, column): last column integer / fractional, the column before it, before the first column; same for rows
            edge = [(ym, ox + WIN_W - 1), (ym, ox + WIN_W - 0.5), (ym, ox + WIN_W - 1.75), (ym, ox - 0.5),
                    (oy + WIN_H - 1, xm), (oy + WIN_H - 0.5, xm), (oy + WIN_H - 1.25, xm), (oy - 0.5, xm + 0.25)]
            for s, (yy, xx) in zip(slots, edge):
                if -1 < yy < H and -1 < xx < W:
                    th.flat[s], tw.flat[s] = yy, xx
            if _origin(np.floor(th).astype(np.int64).ravel(), np.floor(tw).astype(np.int64).ravel(), th.size) == (ox, oy):
                break
