"""Host-side mirror of the reference's operator API (upsnet/operators/modules/*, upsnet/nms/nms.py)
on top of the sm_90a C ABI.  Same class names, constructor arguments, parameter names/shapes
(so reference checkpoints load) and forward signatures; all compute is in libupsnet_b200.so.

Reference interfaces mirrored (paths relative to /root/reference/upsnet/):
  DeformConv, DeformConvWithOffset      operators/modules/deform_conv.py:27-78
  ModDeformConv(+WithOffsetMask)        operators/modules/mod_deform_conv.py:24-81  (exported as
                                        ModulatedDeformConv too, the name BASELINE.json uses)
  RoIAlign / RoIAlignFunction           operators/modules/roialign.py:20-29, functions/roialign.py:21-43
  FPNRoIAlign                           operators/modules/fpn_roi_align.py:22-62
  gpu_nms_wrapper / nms                 nms/nms.py:43-46, nms/gpu_nms.pyx:23-38
  MaskRemoval, SegTerm, PanopticHead    operators/modules/mask_removal.py:23-93,
                                        operators/modules/unary_logits.py:69-105,
                                        models/resnet_upsnet.py:217-247 (F1: no such class there)
Forward only: the inference hot path (SURVEY.md section 8); backward kernels are the training
config and out of this round's scope.
"""
import collections
import ctypes as C
import math

import numpy as np
import torch
import torch.nn as nn
from torch.nn.modules.utils import _pair
from torch.nn.parameter import Parameter

from . import _lib
from ._lib import call, f32c, query_bytes, require_cuda, try_call

# default arithmetic of the convolution tiles; switched by upsnet_b200.set_precision()
_PRECISION = {"conv": _lib.PREC_FP32_SIMT}
# pair-stream deformable convs gather from a shared-memory window into shared-memory A tiles (csrc/dcn_win.cu); maps with fewer
# than min_pixels output pixels keep the global-gather kernel (measured: 0.058 vs 0.048 ms at 32x64, 0.060 vs 0.075 ms at 64x128)
DCN_WINDOW = {"on": True, "min_pixels": 4096}
USE_TMA = {"on": True}     # False forces the cp.async gather kernel where the TMA-fed one would qualify (A/B tests)


def set_precision(name):
    """Default precision of the convolutions, which also fixes how the engine stores its activation stream:
    'fp32': CUDA-core fp32 tiles on fp32 NCHW activations.
    'bf16': single-pass wgmma tiles; activations stored NHWC as bf16 (half the HBM traffic of fp32).
    'bf16x3': the configuration that meets "fp32 logits within 1e-3"; activations stored NHWC as hi/lo bf16 PAIRS
      (class Pair: same bytes as fp32, ~16 mantissa bits) so that the TMA-fed wgmma kernel runs the three-term split
      (hi*hi + lo*hi + hi*lo) without gather threads.
    An explicit precision= on conv2d / deform_conv changes the arithmetic of that call only, not the stream format."""
    _PRECISION["conv"] = {"fp32": _lib.PREC_FP32_SIMT, "bf16x3": _lib.PREC_BF16X3, "bf16": _lib.PREC_BF16}[name]


def _stream():
    """Storage format of the engine's activation stream under the global precision: 'f32', 'bf16' or 'pair'."""
    return {_lib.PREC_BF16: "bf16", _lib.PREC_BF16X3: "pair"}.get(_PRECISION["conv"], "f32")


class Pair:
    """An activation stored as a hi/lo bf16 pair: `store` is bf16 [N,H,W,2C] (NHWC), channels [0,C) = bf16(v) and
    [C,2C) = bf16(v - hi); v = hi + lo is exact in fp32 (UPSNET_DTYPE_PAIR in include/upsnet_b200.h).  Quacks like the
    logical [N,C,H,W] tensor for the few attributes the engine's module code reads."""
    __slots__ = ("store",)
    dtype = "pair"

    def __init__(self, store):
        assert store.dtype == torch.bfloat16 and store.dim() == 4 and store.shape[-1] % 2 == 0 and store.is_contiguous()
        self.store = store

    @staticmethod
    def from_float(x):
        """x: logical [N,C,H,W] float tensor (any memory format) -> Pair."""
        xs = x.float().permute(0, 2, 3, 1)
        hi = xs.to(torch.bfloat16)
        lo = (xs - hi.float()).to(torch.bfloat16)
        return Pair(torch.cat([hi, lo], dim=-1).contiguous())

    @property
    def shape(self):
        n, h, w, c2 = self.store.shape
        return torch.Size((n, c2 // 2, h, w))

    @property
    def device(self):
        return self.store.device

    @property
    def is_cuda(self):
        return self.store.is_cuda

    def dim(self):
        return 4

    def size(self, i=None):
        return self.shape if i is None else self.shape[i]

    def float(self):
        """fp32 logical [N,C,H,W] (channels_last storage) = hi + lo."""
        c = self.store.shape[-1] // 2
        return (self.store[..., :c].float() + self.store[..., c:].float()).permute(0, 3, 1, 2)

    def record_stream(self, s):
        self.store.record_stream(s)

    def subsample2(self):
        """x[:, :, ::2, ::2] (nn.MaxPool2d(kernel_size=1, stride=2): models/fpn.py:75)."""
        return Pair(self.store[:, ::2, ::2, :].contiguous())


def subsample2(x):
    return x.subsample2() if isinstance(x, Pair) else x[:, :, ::2, ::2].contiguous()


def as_float(x):
    """A Pair becomes its fp32 tensor (hi + lo); plain tensors pass through untouched (no dtype round trip)."""
    return x.float() if isinstance(x, Pair) else x


# launch accounting (bench.py reports gpu_launches) and optional per-call CUDA-event timing of the
# kernels behind one C-ABI call (bench.py's roofline leg; off in normal operation)
STATS = {"launches": 0, "trace": None}


class _Timed:
    """with _Timed(kind, n_kernels, work, device): <C-ABI call> -- counts launches; when
    STATS["trace"] is a list also brackets the call with events on the current stream."""

    def __init__(self, kind, n_kernels, work, device):
        self.kind, self.n, self.work, self.device = kind, n_kernels, work, device
        self.ev = None

    def __enter__(self):
        STATS["launches"] += self.n
        if STATS["trace"] is not None:
            self.ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self.ev[0].record(torch.cuda.current_stream(self.device))
        return self

    def __exit__(self, *exc):
        if self.ev is not None:
            self.ev[1].record(torch.cuda.current_stream(self.device))
            STATS["trace"].append((self.kind, self.ev[0], self.ev[1], self.work))
        return False


def _conv_out(n, pad, dil, k, stride):
    return (n + 2 * pad - (dil * (k - 1) + 1)) // stride + 1


# ------------------------------------------------------------------------------------------------
# tensor-core (wgmma) path plumbing: NHWC views and the packed-weight cache
# ------------------------------------------------------------------------------------------------
def _nhwc(x):
    """[N,C,H,W] logical tensor -> contiguous [N,H,W,C] storage (no copy if already channels_last)."""
    xp = x.permute(0, 2, 3, 1)
    return xp if xp.is_contiguous() else xp.contiguous()


import weakref


def _per_weight(cache, weight, make, device=None, versioned=True):
    """make() once per weight tensor, kept in `cache` (made by _weight_cache): id(tensor) -> (weakref to the tensor,
    version, value).  Keyed on the weight TENSOR OBJECT (weak): a data_ptr key would alias a freed weight whose storage
    the caching allocator handed to a new tensor.  Entries die with their tensor; with `versioned`, _version catches
    in-place updates; with `device`, a value (None allowed) made for another device is made again."""
    hit = cache.get(id(weight))
    if (hit is not None and hit[0]() is weight and (not versioned or hit[1] == weight._version) and
            (device is None or hit[2] is None or hit[2].device == device)):
        return hit[2]
    value = make()
    wid = id(weight)
    cache[wid] = (weakref.ref(weight, lambda _r, _k=wid: cache.pop(_k, None)), weight._version, value)
    return value


_weight_caches = []


def _weight_cache():
    """A new cache for _per_weight, recorded so that forget_packed reaches it."""
    cache = {}
    _weight_caches.append(cache)
    return cache


def forget_packed(tensors):
    """Drop what every per-weight cache holds for `tensors`; it is made again, once, on next use.  The version check
    misses writes that bypass the tensor's version counter, such as an optimiser step replayed from a CUDA graph, so
    a model forgets its parameters wherever they may have changed that way."""
    ids = [id(t) for t in tensors]
    for cache in _weight_caches:
        for i in ids:
            cache.pop(i, None)


def _packed(cache, weight, pack, nbytes, nbytes_args, unsupported=False):
    """upsnet_<pack> of the fp32 weight [Cout,Cin,kh,kw] into a uint8 buffer of upsnet_<nbytes>(*nbytes_args) bytes, made
    once per weight tensor and kept in `cache` (_per_weight).  With `unsupported`, None (cached too) when the size query
    answers UPSNET_E_UNSUPPORTED."""
    def make():
        n = query_bytes(nbytes, *nbytes_args, unsupported=unsupported)
        if n is None:
            return None
        buf = torch.empty(n, dtype=torch.uint8, device=weight.device)
        call(pack, weight.device, f32c(weight.detach()), *weight.shape, buf)
        STATS["launches"] += 1
        return buf
    return _per_weight(cache, weight, make, device=weight.device)


_packed_cache = _weight_cache()


def _packed_weight(weight):
    """bf16 hi/lo planes [Cout_pad][kh*kw][Cin] (upsnet_igemm_pack_weight), cached per weight tensor+version."""
    return _packed(_packed_cache, weight, "igemm_pack_weight", "igemm_packed_weight_bytes", weight.shape)


_dcn_packed_cache = _weight_cache()


def _packed_weight_dcn(weight):
    """upsnet_dcn_pack_weight: bf16 hi/lo planes in the window kernel's K order (16-channel sub-chunk, tap, channel);
    None when the layer shape is not supported by that kernel (cached too).  Cached like _packed_weight."""
    return _packed(_dcn_packed_cache, weight, "dcn_pack_weight", "dcn_packed_weight_bytes", weight.shape, unsupported=True)


def _dcn_window(x, offset, mask, weight, bias, padding, dilation, relu):
    """upsnet_dcn_pair_forward (csrc/dcn_win.cu): Pair in, Pair out, 3x3 / stride 1.  Returns None when the layer does
    not qualify (the caller then takes upsnet_igemm_forward)."""
    N, Cin, H, W = x.shape
    if N * H * W < DCN_WINDOW["min_pixels"]:
        return None
    packed = _packed_weight_dcn(weight)
    if packed is None:
        return None
    Cout, _, kh, kw = weight.shape
    ph, pw = padding; dh, dw = dilation
    Ho, Wo = _conv_out(H, ph, dh, kh, 1), _conv_out(W, pw, dw, kw, 1)
    store = torch.empty((N, Ho, Wo, 2 * Cout), device=x.device, dtype=torch.bfloat16)
    work = {"flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw * 3, "algo_flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw,
            "shape": "N%d %dx%d Cin%d->Cout%d k%d s1 pair->pair (window)" % (N, H, W, Cin, Cout, kh),
            "bytes": float(x.store.numel() * 2 + 4 * weight.numel() + store.numel() * 2 + offset.numel() * 4)}
    with _Timed("dcn", 1, work, x.device):
        rc = try_call("dcn_pair_forward", x.device, x.store, offset, mask, packed, bias, store, N, H, W, Cin, Cout, kh, kw,
                      ph, pw, dh, dw, _lib.EPI_RELU if relu else 0)
    return None if rc == _lib.E_UNSUPPORTED else Pair(store)


_stem_cache = _weight_cache()   # packed bf16 [Cout][kh][8][8] per weight
_stem_ws = None


def stem_conv(x, weight, bias, padding, relu=True, pair=False):
    """k x k / stride-2 convolution of a tiny-Cin fp32 NCHW image (models/resnet.py:155-162 conv1) on the TMA kernel:
    the image is packed to a zero-padded bf16 NHWC8 copy whose 5-D tensor-map boxes are the im2col tiles.
    -> bf16 channels_last activation [N,Cout,Ho,Wo]; pair=True (precision bf16x3): hi and lo copies of the image, three MMAs
    per k-slice, -> Pair.  Raises UpsnetError(UNSUPPORTED) if the driver rejects the map."""
    global _stem_ws
    require_cuda(x, weight, bias)
    x = f32c(x)
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = weight.shape
    dev = x.device

    packed = _packed(_stem_cache, weight, "stem_pack_weight", "stem_packed_weight_bytes", (Cout, kh))
    nb = query_bytes("stem_workspace_bytes", N, H, W, kh, kw, int(padding))
    if _stem_ws is None:
        _stem_ws = _Workspace()
    ws = _stem_ws.get(dev, nb)
    Ho, Wo = (H + 2 * padding - kh) // 2 + 1, (W + 2 * padding - kw) // 2 + 1
    store = torch.empty((N, Ho, Wo, Cout * (2 if pair else 1)), dtype=torch.bfloat16, device=dev)
    fl = 2.0 * N * Ho * Wo * Cout * Cin * kh * kw
    work = {"flops": fl * (3 if pair else 1), "algo_flops": fl,
            "shape": "N%d %dx%d Cin%d->Cout%d k%d s2 float32->%s (stem, TMA)" % (N, H, W, Cin, Cout, kh, "pair" if pair else "bfloat16"),
            "bytes": float(4 * x.numel() + 2 * store.numel())}
    with _Timed("conv2d", 2, work, dev):
        call("stem_forward", dev, x, packed, None if bias is None else f32c(bias), store, N, Cin, H, W,
             Cout, kh, kw, int(padding), (_lib.EPI_RELU if relu else 0) | (_lib.EPI_STEM_PAIR if pair else 0),
             ws, ws.numel())
    return Pair(store) if pair else store.permute(0, 3, 1, 2)


def _tc_ok(Cin, kh, kw, dg, deform=False):
    return (Cin % 64 == 0 or (Cin <= 8 and not deform)) and dg == 1 and kh * kw <= 49


def _count(n_dev):
    """A device-side count argument: None, or an int32 CUDA scalar (read by the kernels, never by the host)."""
    if n_dev is not None:
        assert n_dev.dtype == torch.int32 and n_dev.is_cuda and n_dev.numel() == 1
    return n_dev


def _igemm_tc(kind, x, offset, mask, weight, bias, residual, stride, padding, dilation, relu, prec, out_format,
              out_dtype=None, residual_up2=False, pair_group=0, sigmoid_from=None, n_dev=None):
    """upsnet_igemm_forward: x logical NCHW (any memory format; fp32 or bf16) or a Pair; result logical NCHW whose
    storage is NHWC (channels_last view, the engine layout) unless out_format == 'nchw'.
    Output: bf16 / a Pair when the engine's activation stream (_stream()) is bf16 / pairs and the
    result stays in that NHWC stream; fp32 for plane-wise (NCHW) head outputs or when asked via out_dtype.
    pair_group=G (Pair output only): channels are written as [hi G][lo G] groups and the result is returned as the Pair
    of logical shape [N, G, Ho, Wo*Cout/G] that this storage also is (see MaskBranch).
    n_dev: optional int32 device scalar; images >= n_dev are not computed by the TMA-fed path (their output is unspecified)."""
    sh, sw = stride; ph, pw = padding; dh, dw = dilation
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = weight.shape
    Ho, Wo = _conv_out(H, ph, dh, kh, sh), _conv_out(W, pw, dw, kw, sw)
    nhwc_out = out_format != "nchw"
    x3 = prec == _lib.PREC_BF16X3
    stream = _stream()
    pair_in = isinstance(x, Pair)
    if pair_in:
        assert x3, "Pair activations belong to precision bf16x3"
    elif x3 and stream == "pair" and Cin % 64 == 0:
        x = Pair.from_float(x)                               # entry into the pair stream (API-level callers)
        pair_in = True
    elif x3 and x.dtype != torch.float32:
        x = x.float()                                        # the in-kernel hi/lo split needs fp32 activations
    elif x.dtype not in (torch.float32, torch.bfloat16):
        x = x.float()
    dev = x.device
    pair_out = False
    if out_dtype is None:
        if x3 and stream == "pair" and nhwc_out and Cout % 8 == 0:
            pair_out = True
        else:
            out_dtype = torch.bfloat16 if (stream == "bf16" and prec == _lib.PREC_BF16 and nhwc_out) else torch.float32
    elif out_dtype == "pair":
        pair_out = True
    if pair_in:
        xs, x_dt = x.store, _lib.DTYPE_PAIR
    else:
        xs = f32c(x) if Cin % 64 else _nhwc(x)      # tiny-Cin (stem) mode reads the NCHW fp32 image directly
        x_dt = _lib.DTYPE_BF16 if xs.dtype == torch.bfloat16 else _lib.DTYPE_F32
    packed = _packed_weight(weight)
    if pair_out:
        assert nhwc_out
        store = torch.empty((N, Ho, Wo, 2 * Cout), device=dev, dtype=torch.bfloat16)
        res = None
        if residual is not None:
            res = (residual if isinstance(residual, Pair) else Pair.from_float(residual)).store
        y_dt = _lib.DTYPE_PAIR
    elif nhwc_out:
        store = torch.empty((N, Ho, Wo, Cout), device=dev, dtype=out_dtype)
        res = None if residual is None else _nhwc(as_float(residual).to(out_dtype))
        y_dt = _lib.DTYPE_BF16 if out_dtype == torch.bfloat16 else _lib.DTYPE_F32
    else:
        store = torch.empty((N, Cout, Ho, Wo), device=dev, dtype=out_dtype)
        res = None if residual is None else as_float(residual).to(out_dtype).contiguous()
        y_dt = _lib.DTYPE_BF16 if out_dtype == torch.bfloat16 else _lib.DTYPE_F32
    xbytes = xs.numel() * xs.element_size()
    work = {"flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw * (3 if x3 else 1),
            "algo_flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw,
            "shape": "N%d %dx%d Cin%d->Cout%d k%d s%d %s->%s%s" % (N, H, W, Cin, Cout, kh, sh, "pair" if pair_in else str(xs.dtype)[6:],
                                                              "pair" if pair_out else str(out_dtype)[6:],
                                                              " +res" if residual is not None else ""),
            "bytes": float(xbytes + 4 * weight.numel() +
                           store.numel() * store.element_size() * (2 if residual is not None else 1))}
    flags = (_lib.EPI_RELU if relu else 0) | (_lib.EPI_RES_UP2 if residual_up2 else 0) | \
            (0 if USE_TMA["on"] else _lib.EPI_NO_TMA)
    if pair_group:
        assert pair_out and pair_group % 64 == 0 and Cout % pair_group == 0
        flags |= (pair_group // 64) << 8
    if sigmoid_from is not None:
        assert not pair_out and not nhwc_out and residual is None, "sigmoid epilogue: fp32 NCHW head outputs"
        flags |= _lib.EPI_SIGMOID_FROM(sigmoid_from)
    with _Timed(kind, 1, work, dev):
        call("igemm_forward", dev, xs, offset, mask, packed, bias, res,
             store, N, H, W, Cin, Cout, kh, kw, sh, sw, ph, pw, dh, dw,
             _lib.LAYOUT_NHWC if nhwc_out else _lib.LAYOUT_NCHW, x_dt, y_dt, flags,
             prec, _count(n_dev))
    if pair_out:
        if pair_group:
            return Pair(store.view(N, Ho, Wo * (Cout // pair_group), 2 * pair_group))
        return Pair(store)
    return store.permute(0, 3, 1, 2) if nhwc_out else store


# ------------------------------------------------------------------------------------------------
# functional layer
# ------------------------------------------------------------------------------------------------
def conv2d(x, weight, bias=None, stride=1, padding=0, dilation=1, residual=None, relu=False, precision=None,
           out_format=None, out_dtype=None, residual_up2=False, pair_group=0, sigmoid_from=None, n_dev=None):
    """Dense conv + fused bias / residual / ReLU epilogue.  fp32 precision -> upsnet_conv2d_forward
    (NCHW CUDA-core tiles); bf16x3 / bf16 -> upsnet_igemm_forward (wgmma tiles, NHWC storage).
    n_dev: optional int32 device scalar -- only images < n_dev are needed; the output of the others is unspecified."""
    require_cuda(x, weight, bias, residual)
    prec = _PRECISION["conv"] if precision is None else precision
    if prec != _lib.PREC_FP32_SIMT and _tc_ok(weight.shape[1], weight.shape[2], weight.shape[3], 1):
        if residual_up2 and out_format == "nchw":
            residual, residual_up2 = torch.nn.functional.interpolate(as_float(residual), scale_factor=2, mode="nearest"), False
        return _igemm_tc("conv2d", x, None, None, weight, None if bias is None else f32c(bias), residual,
                         _pair(stride), _pair(padding), _pair(dilation), relu, prec, out_format, out_dtype,
                         residual_up2, pair_group, sigmoid_from, n_dev)
    if sigmoid_from is not None:      # CUDA-core path: the conv entry has no sigmoid epilogue
        y = conv2d(x, weight, bias, stride, padding, dilation, residual, relu, precision, out_format, out_dtype, residual_up2)
        y[:, sigmoid_from:] = torch.sigmoid(y[:, sigmoid_from:])
        return y
    if isinstance(x, Pair):
        x = x.float()
    if isinstance(residual, Pair):
        residual = residual.float()
    if residual_up2:   # CUDA-core path: materialise the nearest-neighbour upsampling (models/fpn.py:33-34)
        residual = torch.nn.functional.interpolate(residual, scale_factor=2, mode="nearest")
    x, weight = f32c(x), f32c(weight)
    bias = None if bias is None else f32c(bias)
    residual = None if residual is None else f32c(residual)
    sh, sw = _pair(stride); ph, pw = _pair(padding); dh, dw = _pair(dilation)
    N, Cin, H, W = x.shape
    Cout, Cin_w, kh, kw = weight.shape
    assert Cin_w == Cin, "groups != 1 is not supported"
    Ho, Wo = _conv_out(H, ph, dh, kh, sh), _conv_out(W, pw, dw, kw, sw)
    y = torch.empty((N, Cout, Ho, Wo), device=x.device, dtype=torch.float32)
    if residual is not None:
        assert residual.shape == y.shape
    prec = _lib.PREC_FP32_SIMT
    work = {"flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw, "algo_flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw,
            "bytes": 4.0 * (x.numel() + weight.numel() + y.numel() * (2 if residual is not None else 1))}
    with _Timed("conv2d_simt", 1, work, x.device):
        call("conv2d_forward", x.device, x, weight, bias, residual, y, N, Cin, H, W,
             Cout, kh, kw, sh, sw, ph, pw, dh, dw, _lib.EPI_RELU if relu else 0, prec)
    return y


def linear(x, weight, bias=None, relu=False, precision=None, out_dtype=None):
    """y = x @ weight.T + bias as a 1x1 convolution over N 'images' of 1x1 pixels.  x: [N,K] tensor, or a Pair of
    logical shape [N,K,1,1] (then the result is a Pair too unless out_dtype says otherwise)."""
    if isinstance(x, Pair):
        y = conv2d(x, _as_1x1(weight), bias, relu=relu, precision=precision, out_dtype=out_dtype)
        return y if isinstance(y, Pair) else y.reshape(y.shape[0], weight.shape[0])
    N, K = x.shape
    y = conv2d(x.reshape(N, K, 1, 1), _as_1x1(weight), bias, relu=relu, precision=precision, out_dtype=out_dtype)
    return y if isinstance(y, Pair) else y.reshape(N, weight.shape[0])


_view_cache = _weight_cache()


def _as_1x1(weight):
    """[Cout,K] -> [Cout,K,1,1] view, cached per weight tensor so the packed-weight cache (keyed on tensor
    identity) hits on every call."""
    return _per_weight(_view_cache, weight, lambda: weight.reshape(weight.shape[0], weight.shape[1], 1, 1), versioned=False)


def deform_conv(data, offset, weight, bias=None, stride=1, padding=0, dilation=1, deformable_groups=1,
                mask=None, relu=False, precision=None, out_format=None, out_dtype=None):
    """DeformConvFunction.forward (functions/deform_conv.py:26-57); with `mask` (already 2*sigmoid)
    ModDeformConvFunction.forward (functions/mod_deform_conv.py:25-59).  One fused launch."""
    require_cuda(data, offset, weight, bias, mask)
    prec = _PRECISION["conv"] if precision is None else precision
    use_tc = prec != _lib.PREC_FP32_SIMT and _tc_ok(weight.shape[1], weight.shape[2], weight.shape[3], deformable_groups, True)
    offset = f32c(offset)
    bias = None if bias is None else f32c(bias)
    mask = None if mask is None else f32c(mask)
    sh, sw = _pair(stride); ph, pw = _pair(padding); dh, dw = _pair(dilation)
    if use_tc:
        N, Cin, H, W = data.shape
        kh, kw = weight.shape[2], weight.shape[3]
        Ho, Wo = _conv_out(H, ph, dh, kh, sh), _conv_out(W, pw, dw, kw, sw)
        assert tuple(offset.shape) == (N, 2 * kh * kw, Ho, Wo), offset.shape
        if mask is not None:
            assert tuple(mask.shape) == (N, kh * kw, Ho, Wo), mask.shape
        if (DCN_WINDOW["on"] and isinstance(data, Pair) and prec == _lib.PREC_BF16X3 and (sh, sw) == (1, 1) and
                out_format != "nchw" and out_dtype in (None, "pair") and _stream() == "pair"):
            y = _dcn_window(data, offset, mask, weight, bias, (ph, pw), (dh, dw), relu)
            if y is not None:
                return y
        return _igemm_tc("dcn", data, offset, mask, weight, bias, None, (sh, sw), (ph, pw), (dh, dw), relu, prec,
                         out_format, out_dtype)
    data, weight = f32c(as_float(data)), f32c(weight)
    N, Cin, H, W = data.shape
    Cout, Cin_w, kh, kw = weight.shape
    assert Cin_w == Cin, "groups != 1 is not supported (the reference ignores `groups`)"
    Ho, Wo = _conv_out(H, ph, dh, kh, sh), _conv_out(W, pw, dw, kw, sw)
    assert tuple(offset.shape) == (N, 2 * kh * kw * deformable_groups, Ho, Wo), offset.shape
    if mask is not None:
        assert tuple(mask.shape) == (N, kh * kw * deformable_groups, Ho, Wo), mask.shape
    y = torch.empty((N, Cout, Ho, Wo), device=data.device, dtype=torch.float32)
    prec = _lib.PREC_FP32_SIMT
    work = {"flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw, "algo_flops": 2.0 * N * Ho * Wo * Cout * Cin * kh * kw,
            "bytes": 4.0 * (data.numel() + offset.numel() + weight.numel() + y.numel() +
                            (mask.numel() if mask is not None else 0))}
    with _Timed("dcn_simt", 1, work, data.device):
        call("dcn_forward", data.device, data, offset, mask, weight, bias, y, N, Cin,
             H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, deformable_groups,
             _lib.EPI_RELU if relu else 0, prec)
    return y


def roi_align(features, rois, pooled_height, pooled_width, spatial_scale, sampling_ratio=2, layout="nchw"):
    require_cuda(features, rois)
    features, rois = f32c(features), f32c(rois)
    assert rois.dim() == 2 and rois.shape[1] == 5
    R = rois.shape[0]
    if layout == "nchw":
        B, Cc, H, W = features.shape
        out = torch.empty((R, Cc, pooled_height, pooled_width), device=features.device, dtype=torch.float32)
        lay = _lib.LAYOUT_NCHW
    else:
        B, H, W, Cc = features.shape
        out = torch.empty((R, pooled_height, pooled_width, Cc), device=features.device, dtype=torch.float32)
        lay = _lib.LAYOUT_NHWC
    if R == 0:
        return out
    with _Timed("roi_align", 1, {"bytes": 4.0 * out.numel()}, features.device):
        call("roi_align_forward", features.device, features, B, Cc, H, W, lay, 0, rois, R, pooled_height,
             pooled_width, sampling_ratio, float(spatial_scale), out)
    return out


def max_pool2d(x, kernel_size, stride, padding):
    """nn.MaxPool2d on the engine's activation stream (models/resnet.py:163).  x is a logical NCHW tensor; the
    kernel works on NHWC storage (channels_last tensors are used as they are) in bf16 or fp32."""
    require_cuda(x)
    N, Cc, H, W = x.shape
    Ho = (H + 2 * padding - kernel_size) // stride + 1
    Wo = (W + 2 * padding - kernel_size) // stride + 1
    if isinstance(x, Pair):
        store = torch.empty((N, Ho, Wo, 2 * Cc), device=x.device, dtype=torch.bfloat16)
        with _Timed("maxpool", 1, {"bytes": float((x.store.numel() + store.numel()) * 2)}, x.device):
            call("maxpool2d_nhwc", x.device, x.store, store, N, H, W, Cc, kernel_size, stride, padding, _lib.DTYPE_PAIR)
        return Pair(store)
    if x.dtype not in (torch.float32, torch.bfloat16):
        x = x.float()
    xs = _nhwc(x)
    store = torch.empty((N, Ho, Wo, Cc), device=x.device, dtype=x.dtype)
    with _Timed("maxpool", 1, {"bytes": float((xs.numel() + store.numel()) * x.element_size())}, x.device):
        call("maxpool2d_nhwc", x.device, xs, store, N, H, W, Cc, kernel_size, stride, padding,
             1 if x.dtype == torch.bfloat16 else 0)
    return store.permute(0, 3, 1, 2)


def upsample_bilinear(x, factor):
    """nn.Upsample(scale_factor=factor, mode='bilinear', align_corners=False) on contiguous NCHW fp32 planes
    (models/fcn.py:88-101: the semantic logits)."""
    require_cuda(x)
    x = f32c(x)
    N, Cc, H, W = x.shape
    y = torch.empty((N, Cc, H * factor, W * factor), dtype=torch.float32, device=x.device)
    with _Timed("upsample", 1, {"bytes": 4.0 * (x.numel() + y.numel())}, x.device):
        call("upsample_bilinear_nchw", x.device, x, y, N * Cc, H, W, int(factor))
    return y


def upsample2_bilinear(x):
    """F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False) on the activation stream (models/fpn.py:27-35,
    network.fpn_upsample_method = 'bilinear'): x a Pair, or a bf16 / fp32 logical [N,C,h,w] tensor (NHWC storage; a
    copy only when it is not channels_last) -> [N,C,2h,2w] in x's format, interpolated in fp32 and rounded once."""
    require_cuda(x)
    N, Cc, h, w = x.shape
    xs, dt = _gn_store(x)
    y = torch.empty((N, 2 * h, 2 * w, xs.shape[-1]), dtype=xs.dtype, device=xs.device)
    work = {"bytes": float((xs.numel() + y.numel()) * xs.element_size()),
            "shape": "N%d %dx%d C%d %s" % (N, h, w, Cc, {0: "float32", 1: "bfloat16", 2: "pair"}[dt])}
    with _Timed("upsample2_bilinear", 1, work, xs.device):
        call("upsample2_bilinear_nhwc", xs.device, xs, y, N, h, w, Cc, dt)
    return _gn_wrap(y, dt)


def fcn_score_fuse(s2, s3, s4, s5):
    """s2 + up2(s3) + up4(s4) + up8(s5) on contiguous NCHW fp32 score maps (models/fcn.py:94-101 after the engine's
    score-before-upsample rewrite), one launch instead of three F.interpolate + three adds."""
    require_cuda(s2, s3, s4, s5)
    s2, s3, s4, s5 = f32c(s2), f32c(s3), f32c(s4), f32c(s5)
    N, Cc, H, W = s2.shape
    assert s3.shape == (N, Cc, H // 2, W // 2) and s4.shape == (N, Cc, H // 4, W // 4) and s5.shape == (N, Cc, H // 8, W // 8)
    out = torch.empty_like(s2)
    with _Timed("upsample", 1, {"bytes": 4.0 * (2 * s2.numel() + s3.numel() + s4.numel() + s5.numel())}, s2.device):
        call("fcn_score_fuse", s2.device, s2, s3, s4, s5, out, N * Cc, H, W)
    return out


def _gn_store(x, like=None):
    """(NHWC storage, dtype code) of an activation for the GroupNorm kernels: a Pair's store, or the NHWC storage of a
    bf16 / fp32 logical [N,C,H,W] tensor (a copy only when it is not channels_last).  With `like`, x is first brought
    to the format of that storage (the residual of the FPN top-down add)."""
    if like is not None:
        if like.dtype == "pair":
            x = x if isinstance(x, Pair) else Pair.from_float(x)
        else:
            x = as_float(x).to(like.dtype)
    if isinstance(x, Pair):
        return x.store, _lib.DTYPE_PAIR
    if x.dtype not in (torch.float32, torch.bfloat16):
        x = x.float()
    return _nhwc(x), (_lib.DTYPE_BF16 if x.dtype == torch.bfloat16 else _lib.DTYPE_F32)


def _gn_wrap(store, dt):
    return Pair(store) if dt == _lib.DTYPE_PAIR else store.permute(0, 3, 1, 2)


def group_norm(x, weight, bias, groups=32, eps=1e-5, relu=False, residual=None, residual_up2=False, shift=None,
               return_stats=False, upsample="nearest"):
    """nn.GroupNorm(groups, C) over whole maps, with the optional epilogue y = act(GN(x) + shift + up2(residual)):
    shift float32 [N, C] (FPN's context vector, models/fpn.py:84-86), residual [N,C,H/2,W/2] read with 2x up-sampling
    (the FPN top-down add; residual_up2 must be set), nearest or, with upsample='bilinear', bilinear with
    align_corners=False (network.fpn_upsample_method), ReLU.  x: a Pair, or a bf16 / fp32 logical [N,C,H,W]
    tensor; y has x's format (Pair, or NHWC storage viewed as [N,C,H,W]).  With return_stats also the float32
    [N, groups, 2] (mean, 1 / sqrt(var + eps)) that upsnet_group_norm_backward reads."""
    require_cuda(x, weight, bias, shift)
    if (residual is not None) != bool(residual_up2):
        raise _lib.UpsnetError("group_norm: a residual is read with 2x up-sampling only (residual_up2=True)")
    if upsample not in ("nearest", "bilinear"):
        raise _lib.UpsnetError("group_norm: upsample %r is not one of 'nearest', 'bilinear'" % (upsample,))
    N, C, H, W = x.shape
    xs, dt = _gn_store(x)
    res = None if residual is None else _gn_store(residual, like=xs if dt != _lib.DTYPE_PAIR else x)[0]
    y = torch.empty_like(xs)
    stats = torch.empty((N, groups, 2), dtype=torch.float32, device=xs.device)
    ws = torch.empty(query_bytes("group_norm_workspace_bytes", N, C, H, W, groups), dtype=torch.uint8, device=xs.device)
    nbytes = xs.numel() * xs.element_size()
    work = {"bytes": float(3 * nbytes + (0 if res is None else res.numel() * res.element_size())),
            "shape": "N%d %dx%d C%d G%d %s%s%s" % (N, H, W, C, groups, {0: "float32", 1: "bfloat16", 2: "pair"}[dt],
                                                  " +res" if res is not None else "", " +shift" if shift is not None else "")}
    flags = (_lib.EPI_RELU if relu else 0) | (_lib.EPI_RES_UP2 if res is not None else 0)
    if res is not None and upsample == "bilinear":
        flags |= _lib.EPI_RES_BILINEAR
        work["shape"] += " bilinear"
    with _Timed("group_norm", 3, work, xs.device):
        call("group_norm_forward", xs.device, xs, f32c(weight), f32c(bias), None if shift is None else f32c(shift), res,
             y, stats, N, C, H, W, groups, float(eps), dt, flags, ws, ws.numel())
    out = _gn_wrap(y, dt)
    return (out, stats) if return_stats else out


def group_norm_rows(x, weight, bias, groups=32, eps=1e-5, relu=False, n_dev=None):
    """nn.GroupNorm(groups, C) of every row on its own, one launch: x a Pair or bf16 / fp32 tensor of logical shape
    [R,C,h,w] (the mask branch's roi maps) or a [R,C] tensor (RCNN fc6, models/rcnn.py:102 views it as [R,C,1,1]).
    n_dev: optional int32 device count; rows >= n_dev are skipped (their output is unspecified).  y has x's format."""
    require_cuda(x, weight, bias)
    flat = not isinstance(x, Pair) and x.dim() == 2
    xs, dt = _gn_store(x.reshape(x.shape[0], x.shape[1], 1, 1) if flat else x)
    R, h, w, _ = xs.shape
    C = weight.shape[0]
    y = torch.empty_like(xs)
    work = {"bytes": float(2 * xs.numel() * xs.element_size()),
            "shape": "R%d %dx%d C%d G%d rows" % (R, h, w, C, groups)}
    with _Timed("group_norm", 1, work, xs.device):
        call("group_norm_rows", xs.device, xs, f32c(weight), f32c(bias), y, R, C, h * w, groups, float(eps), dt,
             _lib.EPI_RELU if relu else 0, _count(n_dev))
    return y.reshape(R, C) if flat else _gn_wrap(y, dt)


def fpn_roi_align(feats, rois, pooled_height, pooled_width, spatial_scales, sampling_ratio=2, layout="nchw",
                  return_levels=False, n_dev=None):
    """FPNRoIAlign.forward in one launch (level assignment on device, output already in roi order).
    n_dev: optional int32 device scalar (pair features only) -- rois >= n_dev are skipped, their output is unspecified."""
    assert len(feats) == 4 and len(spatial_scales) == 4
    require_cuda(rois, *feats)
    rois = f32c(rois)
    R = rois.shape[0]
    if isinstance(feats[0], Pair):
        # hi/lo pair features -> Pair result: [R,C,PH,PW] pair pixels, or (layout 'flat_pair') the [R, PH*PW*C, 1, 1]
        # pair of the flattened (ph, pw, c) roi feature that the RCNN fc6 consumes as a 1x1 'image'
        assert all(isinstance(f, Pair) for f in feats) and layout in ("auto", "nhwc", "flat_pair") and not return_levels
        B, Cc = feats[0].shape[0], feats[0].shape[1]
        flat = layout == "flat_pair"
        if flat:
            out = torch.empty((R, 1, 1, 2 * pooled_height * pooled_width * Cc), device=rois.device, dtype=torch.bfloat16)
        else:
            out = torch.empty((R, pooled_height, pooled_width, 2 * Cc), device=rois.device, dtype=torch.bfloat16)
        if R > 0:
            fp = (C.c_void_p * 4)(*[f.store.data_ptr() for f in feats])
            hs = (C.c_int * 4)(*[f.shape[2] for f in feats]); ws = (C.c_int * 4)(*[f.shape[3] for f in feats])
            sc = (C.c_float * 4)(*[float(s_) for s_ in spatial_scales])
            with _Timed("roi_align_fpn", 1, {"bytes": 2.0 * out.numel()}, rois.device):
                call("roi_align_fpn_forward", rois.device, fp, hs, ws, sc, B, Cc,
                     _lib.LAYOUT_FLAT_PAIR if flat else _lib.LAYOUT_NHWC, _lib.DTYPE_PAIR, rois, R, pooled_height,
                     pooled_width, sampling_ratio, out, None, _count(n_dev))
        return Pair(out)
    if layout == "auto":
        # engine tensors: logical NCHW; if every level is stored channels_last use the NHWC kernel
        # (coalesced channel vectors) and hand back a logical-NCHW view of the NHWC result
        cl = all(f.dim() == 4 and f.permute(0, 2, 3, 1).is_contiguous() and not f.is_contiguous() for f in feats)
        if cl:
            out = fpn_roi_align([f.permute(0, 2, 3, 1) for f in feats], rois, pooled_height, pooled_width,
                                spatial_scales, sampling_ratio, "nhwc", return_levels)
            return (out[0].permute(0, 3, 1, 2), out[1]) if return_levels else out.permute(0, 3, 1, 2)
        layout = "nchw"
    bf16 = layout == "nhwc" and all(f.dtype == torch.bfloat16 for f in feats)
    feats = [f.contiguous() for f in feats] if bf16 else [f32c(f) for f in feats]
    odt = torch.bfloat16 if bf16 else torch.float32
    if layout == "nchw":
        B, Cc = feats[0].shape[0], feats[0].shape[1]
        Hs = [f.shape[2] for f in feats]; Ws = [f.shape[3] for f in feats]
        out = torch.empty((R, Cc, pooled_height, pooled_width), device=rois.device, dtype=torch.float32)
        lay = _lib.LAYOUT_NCHW
    else:
        B, Cc = feats[0].shape[0], feats[0].shape[3]
        Hs = [f.shape[1] for f in feats]; Ws = [f.shape[2] for f in feats]
        out = torch.empty((R, pooled_height, pooled_width, Cc), device=rois.device, dtype=odt)
        lay = _lib.LAYOUT_NHWC
    assert n_dev is None, "fpn_roi_align: the roi count bound is implemented for pair features"
    levels = torch.empty((R,), device=rois.device, dtype=torch.int32) if return_levels else None
    fp = (C.c_void_p * 4)(*[f.data_ptr() for f in feats])
    hs = (C.c_int * 4)(*Hs); ws = (C.c_int * 4)(*Ws)
    sc = (C.c_float * 4)(*[float(s) for s in spatial_scales])
    with _Timed("roi_align_fpn", 1, {"bytes": 4.0 * out.numel()}, rois.device):
        call("roi_align_fpn_forward", rois.device, fp, hs, ws, sc, B, Cc, lay, 1 if bf16 else 0, rois, R, pooled_height,
             pooled_width, sampling_ratio, out, levels, None)
    return (out, levels) if return_levels else out


# ------------------------------------------------------------------------------------------------
# NMS
# ------------------------------------------------------------------------------------------------
import threading


class _WsSlot(threading.local):
    """Engine lane whose scratch buffers the C-ABI calls of THIS THREAD use (model._run_static / PipelinedEngine set it around
    a lane's work).  Thread-local: the reference's thread-per-GPU DataParallel usage (one Python thread per device) must not
    see another thread's lane.  Dict-style access (`WS_SLOT["i"]`) is kept for the callers."""
    i = 0

    def __getitem__(self, k):
        assert k == "i"
        return self.i

    def __setitem__(self, k, v):
        assert k == "i"
        self.i = int(v)


WS_SLOT = _WsSlot()


class _Workspace:
    """Caller-owned, grow-only device scratch (the C ABI never allocates).  A buffer that is outgrown is RETIRED, not
    freed: captured CUDA graphs (model._run_static) have its raw pointer baked in and keep writing to it on replay, so
    handing the block back to the caching allocator would let a replay corrupt whatever tensor reuses it (ADVICE r1).
    Growth is geometric (>= 1.5x), which bounds the retired bytes by about twice the final size."""

    def __init__(self):
        self.buf = {}
        self.retired = []

    def get(self, device, nbytes):
        key = (device, WS_SLOT["i"])     # one scratch set per engine lane: lanes run concurrently on their own streams
        b = self.buf.get(key)
        if b is None or b.numel() < nbytes:
            if b is not None:
                self.retired.append(b)
                nbytes = max(int(nbytes), int(b.numel() * 1.5))
            b = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)
            self.buf[key] = b
        return b


_nms_ws = _Workspace()
_nms_ws_side = _Workspace()   # second scratch buffer: an NMS running concurrently on another stream must not share the first
_pan_ws = _Workspace()


def nms_segmented(boxes_sorted, seg_offsets, max_seg_len, thresh, side=False):
    """boxes_sorted [total,4] fp32 sorted by descending score inside each segment; seg_offsets int32
    [S+1] (device).  Returns (keep [S,max_seg_len] int32 positions relative to segment start,
    counts [S] int32) -- both on the device, no host synchronisation."""
    require_cuda(boxes_sorted, seg_offsets)
    boxes_sorted = f32c(boxes_sorted)
    assert seg_offsets.dtype == torch.int32
    S = seg_offsets.numel() - 1
    dev = boxes_sorted.device
    nbytes = query_bytes("nms_workspace_bytes", S, max_seg_len)
    ws = (_nms_ws_side if side else _nms_ws).get(dev, nbytes)
    keep = torch.empty((S, max_seg_len), dtype=torch.int32, device=dev)
    cnt = torch.empty((S,), dtype=torch.int32, device=dev)
    with _Timed("nms", 2, {"bytes": 20.0 * boxes_sorted.shape[0]}, dev):
        call("nms_segmented", dev, boxes_sorted, seg_offsets, S, max_seg_len, float(thresh), keep, cnt, ws, ws.numel())
    return keep, cnt


def im_info_device(im_info, dev):
    """The image geometry row (h, w, scale) as a float32 [3] tensor on `dev`.  A float32 tensor already there is returned
    as it is; a host row ([3] or [1,3], numpy or tensor) is uploaded through pinned memory without blocking the host
    (torch's pinned allocator keeps the staging block until the copy has run).  The detection kernels read the row when
    they run, so a captured graph that reads a device row takes a new image size by a copy into that row."""
    if torch.is_tensor(im_info) and im_info.device == torch.device(dev) and im_info.dtype == torch.float32:
        assert im_info.numel() == 3, "im_info: one (h, w, scale) row"
        return im_info.reshape(3)
    t = im_info.detach().cpu() if torch.is_tensor(im_info) else torch.from_numpy(np.asarray(im_info, dtype=np.float32))
    t = t.to(torch.float32).reshape(-1)[:3].contiguous()
    if torch.device(dev).type != "cuda":
        return t.to(dev)
    return t.pin_memory().to(dev, non_blocking=True)


def rpn_decode(bbox_preds, top_idx, shapes, strides, base_anchors, A, im_info):
    """Fused anchors + bbox_transform + clip_boxes for the pre-NMS top-k of every level (one launch).
    bbox_preds[l] fp32 [4A,h,w] (contiguous), top_idx[l] int64 [k_l] flat (y,x,a) indices, base_anchors float64
    [L,A,4] on the device, im_info the (h, w, scale) row (CUDA float32 [3], or a host row: im_info_device).
    -> boxes [sum k_l, 4]."""
    L = len(bbox_preds)
    dev = bbox_preds[0].device
    require_cuda(*bbox_preds, *top_idx, base_anchors)
    assert base_anchors.dtype == torch.float64 and base_anchors.is_contiguous()
    bbox_preds = [f32c(b) for b in bbox_preds]
    top_idx = [t.contiguous() for t in top_idx]
    assert all(t.dtype == torch.int64 for t in top_idx)
    info = im_info_device(im_info, dev)
    ks = [int(t.numel()) for t in top_idx]
    out = torch.empty((sum(ks), 4), dtype=torch.float32, device=dev)
    vp, ci = C.c_void_p, C.c_int
    with _Timed("rpn_decode", 1, {"bytes": 56.0 * sum(ks)}, dev):
        call("rpn_decode", dev, (vp * L)(*[b.data_ptr() for b in bbox_preds]), (vp * L)(*[t.data_ptr() for t in top_idx]),
             (ci * L)(*ks), (ci * L)(*[int(s[0]) for s in shapes]), (ci * L)(*[int(s[1]) for s in shapes]),
             (ci * L)(*[int(s) for s in strides]), base_anchors, L, int(A), info, out)
    return out


_topk_ws = None


def rpn_topk(probs, A, pre_nms_top_n):
    """Top pre_nms_top_n anchors of every level in one call.  probs[l] fp32 [A,h,w] -> (scores [sum k_l], flat (y,x,a)
    indices int64 [sum k_l], [k_l]): sorted by descending score, ties by ascending index."""
    global _topk_ws
    L = len(probs)
    dev = probs[0].device
    require_cuda(*probs)
    probs = [f32c(pr) for pr in probs]
    ks = [min(int(pre_nms_top_n), int(pr.numel())) for pr in probs]
    out_s = torch.empty((sum(ks),), dtype=torch.float32, device=dev)
    out_i = torch.empty((sum(ks),), dtype=torch.int64, device=dev)
    if _topk_ws is None:
        _topk_ws = _Workspace()
    nbytes = query_bytes("rpn_topk_workspace_bytes", L)
    ws = _topk_ws.get(dev, nbytes)
    vp, ci = C.c_void_p, C.c_int
    with _Timed("rpn_topk", 7, {"bytes": 4.0 * 6 * sum(pr.numel() for pr in probs)}, dev):
        call("rpn_topk", dev, (vp * L)(*[pr.data_ptr() for pr in probs]), (ci * L)(*[int(pr.shape[-2]) for pr in probs]),
             (ci * L)(*[int(pr.shape[-1]) for pr in probs]), L, int(A), int(pre_nms_top_n),
             out_s, out_i, ws, ws.numel())
    return out_s, out_i, ks


def rpn_collect(keep, cnt, offs, boxes, scores, post_nms_top_n):
    """Fused proposal collect after the per-level NMS -> (rois [post,5], scores [post], valid [post] bool)."""
    require_cuda(keep, cnt, offs, boxes, scores)
    dev = boxes.device
    S, M = keep.shape
    post = int(post_nms_top_n)
    rois = torch.empty((post, 5), dtype=torch.float32, device=dev)
    out_s = torch.empty((post,), dtype=torch.float32, device=dev)
    ok = torch.empty((post,), dtype=torch.bool, device=dev)
    with _Timed("rpn_collect", 1, {"bytes": 28.0 * post}, dev):
        call("rpn_collect", dev, keep, cnt, offs, f32c(boxes), f32c(scores), S, M, post, rois, out_s, ok)
    return rois, out_s, ok


def maskroi_prepare(rois, roi_valid, bbox_delta, cls_prob, class_agnostic, score_thresh, weights, im_info):
    """Fused MaskROI front half -> (sc [n], cls int32 [n], bx [n,4], offs int32 [nseg+1]), n = R*(C-1):
    candidates first in (segment, score desc, index) order, decoded and clipped to the (h, w, scale) row im_info
    (CUDA float32 [3], or a host row: im_info_device)."""
    require_cuda(rois, roi_valid, bbox_delta, cls_prob)
    rois, bbox_delta, cls_prob = f32c(rois), f32c(bbox_delta), f32c(cls_prob)
    assert roi_valid.dtype == torch.bool and roi_valid.is_contiguous()
    R, Cn = cls_prob.shape
    n = R * (Cn - 1)
    dev = rois.device
    nseg = 1 if class_agnostic else Cn - 1
    info = im_info_device(im_info, dev)
    sc = torch.empty((n,), dtype=torch.float32, device=dev)
    cls = torch.empty((n,), dtype=torch.int32, device=dev)
    bx = torch.empty((n, 4), dtype=torch.float32, device=dev)
    offs = torch.empty((nseg + 1,), dtype=torch.int32, device=dev)
    w4 = (C.c_float * 4)(*[float(w) for w in weights])
    with _Timed("maskroi", 1, {"bytes": 4.0 * (rois.numel() + bbox_delta.numel() + cls_prob.numel())}, dev):
        call("maskroi_prepare", dev, rois, roi_valid, bbox_delta, cls_prob, R, Cn,
             1 if class_agnostic else 0, float(score_thresh), w4, info, sc, cls, bx, offs)
    return sc, cls, bx, offs


def maskroi_finish(keep, cnt, offs, sc, cls, bx, top_n, cap):
    """Fused MaskROI back half -> (scores [cap], boxes [cap,5], cls int64 [cap], n int32 device scalar, flags int32 device
    scalar).  flags != 0 means the static buffers truncated what the reference would have kept: bit 0 = more NMS survivors
    than candidate slots, bit 1 = a tie at the top-n threshold larger than the output slack (ADVICE r1)."""
    require_cuda(keep, cnt, offs, sc, cls, bx)
    dev = sc.device
    nseg, M = keep.shape
    out_sc = torch.empty((cap,), dtype=torch.float32, device=dev)
    out_bx = torch.empty((cap, 5), dtype=torch.float32, device=dev)
    out_cls = torch.empty((cap,), dtype=torch.int64, device=dev)
    n_out = torch.empty((2,), dtype=torch.int32, device=dev)
    with _Timed("maskroi", 1, {"bytes": 32.0 * cap}, dev):
        call("maskroi_finish", dev, keep, cnt, offs, sc, cls, bx, nseg, M, int(top_n),
             int(cap), out_sc, out_bx, out_cls, n_out)
    return out_sc, out_bx, out_cls, n_out[0], n_out[1]


def mask_rows(b1, n1, b2, n2):
    """Rows of the mask branch for one image (upsnet_mask_rows): b1 [cap1,5] / n1 detections, b2 [cap2,5] / n2 panoptic
    candidates (counts: int32 device scalars) -> (rows [cap1+cap2,5], u int32 device scalar, pan_row int32 [cap2]).  rows
    holds the detections, then the candidates whose box matches no detection bit for bit; candidate j's logits are row
    pan_row[j] of the branch's output."""
    require_cuda(b1, n1, b2, n2)
    dev = b1.device
    cap1, cap2 = b1.shape[0], b2.shape[0]
    b1, b2 = f32c(b1), f32c(b2)
    rows = torch.empty((cap1 + cap2, 5), dtype=torch.float32, device=dev)
    u = torch.empty((), dtype=torch.int32, device=dev)
    pan_row = torch.empty((cap2,), dtype=torch.int32, device=dev)
    with _Timed("maskroi", 1, {"bytes": 40.0 * (cap1 + cap2)}, dev):
        call("mask_rows", dev, b1, _count(n1), cap1, b2, _count(n2), cap2, rows, u, pan_row)
    return rows, u, pan_row


def nms(boxes, scores, thresh):
    """Device API: boxes [N,4], scores [N] (CUDA) -> int64 indices of kept boxes, descending score
    (== order[keep] of nms/gpu_nms.pyx:32-38).  One D2H of the count only."""
    require_cuda(boxes, scores)
    n = boxes.shape[0]
    if n == 0:
        return torch.empty((0,), dtype=torch.int64, device=boxes.device)
    _, order = torch.sort(scores.float(), descending=True, stable=True)
    seg = torch.tensor([0, n], dtype=torch.int32, device=boxes.device)
    keep, cnt = nms_segmented(boxes.float()[order], seg, n, thresh)
    k = int(cnt.item())
    return order[keep[0, :k].long()]


def gpu_nms(dets, thresh, device_id=0):
    """nms/gpu_nms.pyx:23-38: dets np.float32 [N,5] on the HOST -> list[int]."""
    dets = np.ascontiguousarray(dets, dtype=np.float32)
    if dets.shape[0] == 0:
        return []
    d = torch.from_numpy(dets).to(torch.device("cuda", device_id))
    return nms(d[:, :4], d[:, 4], thresh).cpu().tolist()


def gpu_nms_wrapper(thresh, device_id):
    """nms/nms.py:43-46."""
    def _nms(dets):
        return gpu_nms(dets, thresh, device_id)
    return _nms


# ------------------------------------------------------------------------------------------------
# modules (reference names / signatures / parameter names)
# ------------------------------------------------------------------------------------------------
def _needs_grad(*tensors):
    """True when autograd records and one of the (plain tensor) inputs or parameters requires grad."""
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors)


def _check_dg_for_grad(deformable_groups):
    if deformable_groups != 1:
        raise NotImplementedError("DeformConv / ModDeformConv backward supports deformable_groups=1 only (got %d); run "
                                  "the forward under torch.no_grad() or with parameters that do not require grad"
                                  % deformable_groups)


class DeformConv(nn.Module):
    """operators/modules/deform_conv.py:27-64.  Parameters are created on CUDA like the reference."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__()
        assert in_channels % groups == 0, 'in_channels must be divisible by groups'
        assert out_channels % groups == 0, 'out_channels must be divisible by groups'
        assert out_channels % deformable_groups == 0, 'out_channels must be divisible by deformable groups'
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation = _pair(padding), _pair(dilation)
        self.groups, self.deformable_groups = groups, deformable_groups
        dev = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
        self.weight = Parameter(torch.empty(out_channels, in_channels // groups, *self.kernel_size, device=dev))
        if bias:
            self.bias = Parameter(torch.empty(out_channels, device=dev))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        n = self.in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def forward(self, data, offset):
        if _needs_grad(data, offset, self.weight, self.bias):
            _check_dg_for_grad(self.deformable_groups)
            from .training import DeformConvFunction      # training path: hand-written backward kernels (csrc/backward.cu)
            return DeformConvFunction.apply(data, offset, self.weight, self.bias, self.stride, self.padding, self.dilation)
        return deform_conv(data, offset, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups)


class DeformConvWithOffset(nn.Module):
    """operators/modules/deform_conv.py:67-78 (submodules `conv_offset`, `conv`)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__()
        self.conv_offset = nn.Conv2d(in_channels, kernel_size * kernel_size * 2 * deformable_groups,
                                     kernel_size=3, stride=1, padding=1)
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()
        self.conv = DeformConv(in_channels, out_channels, kernel_size=kernel_size, stride=stride,
                               padding=padding, dilation=dilation, groups=groups,
                               deformable_groups=deformable_groups, bias=bias)

    def forward(self, x):
        if _needs_grad(x, self.conv_offset.weight, self.conv_offset.bias):
            from .training import OffsetConvFunction      # differentiable offsets, same forward
            return self.conv(x, OffsetConvFunction.apply(x, self.conv_offset.weight, self.conv_offset.bias))
        offset = conv2d(x, self.conv_offset.weight, self.conv_offset.bias, 1, 1, 1, out_format="nchw")
        return self.conv(x, offset)


class ModDeformConv(DeformConv):
    """operators/modules/mod_deform_conv.py:24-67: forward(data, offset_mask) with
    offset = cat(chunk0, chunk1), mask = 2*sigmoid(chunk2)."""

    def forward(self, data, offset_mask):
        offset_1, offset_2, mask = torch.chunk(offset_mask, 3, dim=1)
        offset = torch.cat((offset_1, offset_2), dim=1)
        mask = torch.sigmoid(mask) * 2
        if _needs_grad(data, offset_mask, self.weight, self.bias):
            _check_dg_for_grad(self.deformable_groups)
            from .training import ModDeformConvFunction
            return ModDeformConvFunction.apply(data, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation)
        return deform_conv(data, offset, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups, mask=mask)


ModulatedDeformConv = ModDeformConv


class ModDeformConvWithOffsetMask(nn.Module):
    """operators/modules/mod_deform_conv.py:70-81 (submodules `conv_offset_mask`, `conv`)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__()
        self.conv_offset_mask = nn.Conv2d(in_channels, kernel_size * kernel_size * 3 * deformable_groups,
                                          kernel_size=3, stride=1, padding=1)
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()
        self.conv = ModDeformConv(in_channels, out_channels, kernel_size=kernel_size, stride=stride,
                                  padding=padding, dilation=dilation, groups=groups,
                                  deformable_groups=deformable_groups, bias=bias)

    def forward(self, x):
        if _needs_grad(x, self.conv_offset_mask.weight, self.conv_offset_mask.bias):
            from .training import OffsetConvFunction
            return self.conv(x, OffsetConvFunction.apply(x, self.conv_offset_mask.weight, self.conv_offset_mask.bias))
        om = conv2d(x, self.conv_offset_mask.weight, self.conv_offset_mask.bias, 1, 1, 1, out_format="nchw")
        return self.conv(x, om)


class RoIAlignFunction:
    """functions/roialign.py:21-43 call shape: RoIAlignFunction(ph, pw, scale)(features, rois)."""

    def __init__(self, pooled_height, pooled_width, spatial_scale, sampling_ratio=2):
        self.pooled_width, self.pooled_height = int(pooled_width), int(pooled_height)
        self.spatial_scale, self.sampling_ratio = float(spatial_scale), sampling_ratio

    def __call__(self, features, rois):
        if not features.is_cuda:
            raise Exception('not implemented')
        if torch.is_grad_enabled() and features.requires_grad:
            from .training import RoIAlignFunction as _F      # training path: upsnet_roi_align_backward
            return _F.apply(features, rois, self.pooled_height, self.pooled_width, self.spatial_scale, self.sampling_ratio)
        return roi_align(features, rois, self.pooled_height, self.pooled_width, self.spatial_scale,
                         self.sampling_ratio)


class RoIAlign(nn.Module):
    """operators/modules/roialign.py:20-29."""

    def __init__(self, pooled_height, pooled_width, spatial_scale):
        super().__init__()
        self.pooled_width, self.pooled_height = int(pooled_width), int(pooled_height)
        self.spatial_scale = float(spatial_scale)

    def forward(self, features, rois):
        return RoIAlignFunction(self.pooled_height, self.pooled_width, self.spatial_scale)(features, rois)


ROIAlign = RoIAlign


class FPNRoIAlign(nn.Module):
    """operators/modules/fpn_roi_align.py:22-62; forward([P2..P5], rois[N,5]) -> [N,C,ph,pw]."""

    def __init__(self, pooled_height, pooled_width, spatial_scale, with_expand=False):
        super().__init__()
        self.pooled_width, self.pooled_height = int(pooled_width), int(pooled_height)
        self.spatial_scale = spatial_scale
        self.with_expand = with_expand

    def forward(self, feat, rois):
        feat = list(feat)
        if torch.is_grad_enabled() and any(getattr(f, "requires_grad", False) for f in feat):
            if not all(isinstance(f, torch.Tensor) and f.dtype == torch.float32 for f in feat):
                raise TypeError("FPNRoIAlign: the backward kernel takes fp32 features; pair / bf16 features cannot "
                                "require grad")
            from .training import FPNRoIAlignFunction     # training path: upsnet_roi_align_backward per level
            return FPNRoIAlignFunction.apply(rois, self.pooled_height, self.pooled_width, self.spatial_scale, 2, *feat)
        return fpn_roi_align(feat, rois, self.pooled_height, self.pooled_width, self.spatial_scale,
                             layout="auto")


# ------------------------------------------------------------------------------------------------
# panoptic head
# ------------------------------------------------------------------------------------------------
def panoptic_fuse(fcn_output, mask_rois, cls_prob, mask_logit, cls_idx, num_stuff, fraction_threshold=0.3,
                  want_sem=False, n_dev=None, workspace_bytes=None, up4=False):
    """Fused MaskRemoval + SegTerm + void/argmax (upsnet_panoptic_head).
    fcn_output [1,S,H,W]; mask_rois [n,4]; cls_prob [n]; mask_logit [n,1,28,28] or [n,28,28];
    cls_idx int64 [n].  Returns (keep_inds int64 [k], panoptic_output int64 [1,H,W][, sem int64 [1,H,W]]).
    With n_dev (int32 device scalar, actual count <= n) nothing is read back: keep_inds is the padded
    [n] buffer and the device count k is returned as an extra last element (static-shape engine path).
    up4=True: `fcn_output` is the quarter-resolution score map [1,S,H/4,W/4] (FCNHead's 'fcn_score'); its x4 bilinear
    up-sampling (models/fcn.py:88-101) is evaluated inside the kernel, bit-identical to upsample_bilinear(score, 4)."""
    require_cuda(fcn_output, mask_rois, cls_prob, mask_logit, cls_idx)
    assert fcn_output.dim() == 4 and fcn_output.shape[0] == 1, "only support batch size = 1"
    fcn = f32c(fcn_output)
    _, S, H, W = fcn.shape
    if up4:
        Hs, Ws, H, W = H, W, 4 * H, 4 * W
    boxes, prob, ml = f32c(mask_rois), f32c(cls_prob).reshape(-1), f32c(mask_logit)
    cls = cls_idx.to(torch.int64).contiguous()
    n = boxes.shape[0]
    assert boxes.shape == (n, 4) and prob.numel() == n and ml.numel() == n * 784 and cls.numel() == n
    dev = fcn.device
    num_thing = S - num_stuff
    nbytes = query_bytes("panoptic_workspace_bytes", n, H, W, num_thing)
    if workspace_bytes is None:
        ws = _pan_ws.get(dev, nbytes)
    else:
        # caller-chosen (smaller) workspace: the instances' bit windows are then processed in several rounds of
        # consecutive score ranks -- same results (upsnet_panoptic_workspace_min_bytes is the floor)
        ws = torch.empty(int(workspace_bytes), dtype=torch.uint8, device=dev)
    if n_dev is not None:
        assert n_dev.dtype == torch.int32 and n_dev.is_cuda
    keep = torch.zeros((max(n, 1),), dtype=torch.int64, device=dev)
    k = torch.empty((1,), dtype=torch.int32, device=dev)
    labels = torch.empty((1, H, W), dtype=torch.int64, device=dev)
    sem = torch.empty((1, H, W), dtype=torch.int64, device=dev) if want_sem else None
    work = {"bytes": 4.0 * S * H * W / (16 if up4 else 1) + 8.0 * H * W * (2 if want_sem else 1) + n * (4.0 * 784 + 24)}
    with _Timed("panoptic_head", 5, work, dev):
        if up4:
            call("panoptic_head_up4", dev, fcn, S, Hs, Ws, boxes, prob, ml, cls, n, n_dev,
                 num_stuff, float(fraction_threshold), keep, k, labels,
                 sem, ws, ws.numel())
        else:
            call("panoptic_head", dev, fcn, S, H, W, boxes, prob, ml, cls, n, n_dev,
                 num_stuff, float(fraction_threshold), keep, k, labels,
                 sem, ws, ws.numel())
    if n_dev is not None:
        return (keep, labels, sem, k) if want_sem else (keep, labels, k)
    keep = keep[:int(k.item())]
    return (keep, labels, sem) if want_sem else (keep, labels)


class MaskRemoval(nn.Module):
    """operators/modules/mask_removal.py:23-93, same signature and return values:
    forward(mask_rois[n,4], cls_prob[n], mask_prob[n,1,28,28], cls_idx[n], im_shape) ->
    (keep_inds LongTensor [k], mask_energy [1,k,H,W]).  Runs the device kernels of the fused head and, for
    API parity, materialises mask_energy (the fused PanopticHead never does)."""

    def __init__(self, fraction_threshold=0.3):
        super().__init__()
        self.fraction_threshold = fraction_threshold

    def forward(self, mask_rois, cls_prob, mask_prob, cls_idx, im_shape):
        require_cuda(mask_rois, cls_prob, mask_prob, cls_idx)
        boxes, prob, ml = f32c(mask_rois), f32c(cls_prob).reshape(-1), f32c(mask_prob)
        cls = cls_idx.to(torch.int64).contiguous()
        n, (H, W) = boxes.shape[0], (int(im_shape[0]), int(im_shape[1]))
        dev = boxes.device
        num_thing = max(int(cls.max().item()), 1)          # mask_image planes: np.max(cls_idx) (host read, as the reference)
        nbytes = query_bytes("panoptic_workspace_bytes", n, H, W, num_thing)
        ws = _pan_ws.get(dev, nbytes)
        keep = torch.zeros((max(n, 1),), dtype=torch.int64, device=dev)
        k = torch.empty((1,), dtype=torch.int32, device=dev)
        energy = torch.empty((n, H, W), dtype=torch.float32, device=dev)
        with _Timed("mask_removal", 5, {"bytes": 4.0 * n * H * W}, dev):
            call("mask_removal", dev, boxes, prob, ml, cls, n, None, H, W, num_thing,
                 float(self.fraction_threshold), keep, k, energy, ws, ws.numel())
        kk = int(k.item())
        return keep[:kk], energy[:kk].unsqueeze(0)


class SegTerm(nn.Module):
    """operators/modules/unary_logits.py:69-105: (stuff logits view, per-instance boxed copy of the instance's
    thing-class logit).  Pure tensor slicing on the device, same integer conventions as the reference
    (int() truncation, numpy half-to-even round, python-slice clamping).  API parity only: the fused
    PanopticHead evaluates the same windows inside pan_fuse without building [1,k,H,W]."""

    def __init__(self, num_seg_classes, box_scale=1 / 4.0, class_mapping=None, thresh=0.3, num_classes=None):
        super().__init__()
        num_classes = num_classes if num_classes is not None else 9
        self.class_mapping = dict(zip(range(1, num_classes), range(num_seg_classes - num_classes + 1, num_seg_classes))) \
            if class_mapping is None else class_mapping
        self.num_seg_classes, self.num_inst_classes, self.box_scale = num_seg_classes, len(self.class_mapping), box_scale

    def forward(self, cls_indices, seg_score, boxes):
        assert seg_score.shape[0] == 1, "only support batch size = 1"
        cls_np = cls_indices.detach().cpu().numpy()
        seg_energy = seg_score[[0], :-self.num_inst_classes, :, :]
        b = boxes.detach().cpu().numpy()[:, 1:] * self.box_scale
        if cls_np.size == 0:
            return seg_energy, torch.ones_like(seg_energy[[0], [0], :, :]).view(1, 1, seg_energy.shape[2], seg_energy.shape[3]) * -10
        inst = torch.zeros((1, cls_np.shape[0], seg_score.shape[2], seg_score.shape[3]), device=seg_score.device)
        for i in range(cls_np.shape[0]):
            if cls_np[i] == 0:
                continue
            y0, y1 = int(b[i][1]), int(b[i][3].round() + 1)
            x0, x1 = int(b[i][0]), int(b[i][2].round() + 1)
            inst[0, i, y0:y1, x0:x1] = seg_score[0, self.class_mapping[int(cls_np[i])], y0:y1, x0:x1]
        return seg_energy, inst


class MaskTerm(nn.Module):
    """operators/modules/unary_logits.py:24-66 (training twin of MaskRemoval's paste: every roi's 28x28 mask logit is
    bilinearly resized (align_corners=False, ATen rule) to its box at 1/4 scale and pasted into [1,n,h,w]).  Tensor ops
    on the device, differentiable through torch autograd like the reference's F.upsample."""

    def __init__(self, num_seg_classes, box_scale=1 / 4.0, class_mapping=None, num_classes=9, mask_size=28):
        super().__init__()
        self.num_seg_classes, self.box_scale, self.mask_size = num_seg_classes, box_scale, mask_size
        self.class_mapping = dict(zip(range(1, num_classes), range(num_seg_classes - num_classes + 1, num_seg_classes))) \
            if class_mapping is None else class_mapping

    def forward(self, masks, boxes, cls_indices, seg_score):
        assert seg_score.shape[0] == 1, "only support batch size = 1"
        boxes = boxes[:, 1:] * self.box_scale
        H, W = int(seg_score.shape[2]), int(seg_score.shape[3])
        energy = torch.zeros((1, masks.shape[0], H, W), device=seg_score.device)
        ref = boxes.long().tolist()                                          # one host read for all boxes
        for i, (bx0, by0, bx1, by1) in enumerate(ref):
            w, h = max(bx1 - bx0 + 1, 1), max(by1 - by0 + 1, 1)
            m = torch.nn.functional.interpolate(masks[i, 0].view(1, 1, self.mask_size, self.mask_size), size=(h, w),
                                                mode="bilinear", align_corners=False)
            x0, x1, y0, y1 = max(bx0, 0), min(bx1 + 1, W), max(by0, 0), min(by1 + 1, H)
            if x1 > x0 and y1 > y0:
                energy[0, i, y0:y1, x0:x1] = m[0, 0, (y0 - by0):(y1 - by0), (x0 - bx0):(x1 - bx0)]
        return energy


class MaskMatching(nn.Module):
    """operators/modules/mask_matching.py:27-62: panoptic ground truth = stuff labels kept, every (kept) gt instance mask
    painted with its channel index, the rest void (255) or the extra 'unmatched' channel."""

    def __init__(self, num_seg_classes, enable_void, class_mapping=None, num_classes=9):
        super().__init__()
        self.class_mapping = dict(zip(range(1, num_classes), range(num_seg_classes - num_classes + 1, num_seg_classes))) \
            if class_mapping is None else class_mapping
        self.num_seg_classes, self.num_classes = num_seg_classes, num_classes
        self.num_inst_classes, self.enable_void = len(self.class_mapping), enable_void

    def forward(self, gt_segs, gt_masks, keep_inds=None):
        matched = torch.ones_like(gt_segs) * -1
        matched = torch.where(gt_segs <= self.num_seg_classes - self.num_classes, gt_segs, matched)
        matched = torch.where(gt_segs >= 255, gt_segs, matched)
        if keep_inds is not None:
            gt_masks = gt_masks[keep_inds]
        base = self.num_seg_classes - self.num_inst_classes
        for i in range(gt_masks.shape[0]):
            matched[(gt_masks[[i], :, :] != 0) & (gt_masks[[i], :, :] != 255)] = i + base
        matched[matched == -1] = (base + gt_masks.shape[0]) if keep_inds is not None else 255
        return matched


class PanopticHead(nn.Module):
    """The parameter-free panoptic head of models/resnet_upsnet.py:217-247 as one module (the
    reference has no such class: SURVEY.md F1).  forward takes what lines 220-227 consume."""

    def __init__(self, num_seg_classes, num_classes, fraction_threshold=0.3):
        super().__init__()
        self.num_seg_classes, self.num_classes = num_seg_classes, num_classes
        self.num_stuff = num_seg_classes - num_classes + 1  # unary_logits.py:72
        self.fraction_threshold = fraction_threshold

    def forward(self, fcn_output, mask_rois, cls_prob, mask_score, cls_idx, want_sem=False):
        """mask_rois [n,5] (batch,x1,y1,x2,y2) or [n,4]; mask_score [n,1,28,28] = logit of the predicted
        class (resnet_upsnet.py:220).  Returns dict(keep_inds, panoptic_outputs[, fcn_outputs])."""
        boxes = mask_rois[:, 1:] if mask_rois.shape[1] == 5 else mask_rois
        out = panoptic_fuse(fcn_output, boxes, cls_prob, mask_score, cls_idx, self.num_stuff,
                            self.fraction_threshold, want_sem)
        res = {'keep_inds': out[0], 'panoptic_outputs': out[1]}
        if want_sem:
            res['fcn_outputs'] = out[2]
        return res


# ------------------------------------------------------------------------------------------------
# callers either side of the forward (SURVEY section 8f): unified panoptic result, input pipeline
# ------------------------------------------------------------------------------------------------
_uni_ws = _Workspace()


def unified_pan_result(seg, pan, cls_inds, num_seg_classes, num_classes, stuff_area_limit=4 * 64 * 64, k_dev=None,
                       check_errors=True):
    """dataset/base_dataset.py:332-371 get_unified_pan_result for one image, on the device.
    seg / pan: int64 [H,W] or [1,H,W] ('fcn_outputs' / 'panoptic_outputs' of the forward); cls_inds int64 [k]
    ('panoptic_cls_inds').  -> uint8 [H,W,3] (semantic class, instance number, 0).  With check_errors (one int D2H) an
    instance label without a cls_inds entry raises IndexError like the reference."""
    require_cuda(seg, pan, cls_inds)
    seg = seg.reshape(seg.shape[-2:]).to(torch.int64).contiguous()
    pan = pan.reshape(pan.shape[-2:]).to(torch.int64).contiguous()
    cls = cls_inds.to(torch.int64).contiguous()
    H, W = pan.shape
    dev = pan.device
    nb = query_bytes("unified_pan_workspace_bytes", int(num_seg_classes))
    ws = _uni_ws.get(dev, nb)
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
    err = torch.zeros((1,), dtype=torch.int32, device=dev)
    with _Timed("unified_pan", 5, {"bytes": 19.0 * H * W}, dev):
        call("unified_pan_result", dev, seg, pan, cls, int(cls.numel()), k_dev, H, W,
             int(num_seg_classes), int(num_classes), int(stuff_area_limit), out, err,
             ws, ws.numel())
    if check_errors:
        e = int(err.item())
        if e & 2:
            raise IndexError("panoptic label without an entry in cls_inds (base_dataset.py:350)")
        if e & 1:
            raise ValueError("label out of range in seg / pan")
    return out


def prep_image(image_hwc_u8, pixel_means, scale=1.0, stride=32, flip=False, out=None):
    """dataset/base_dataset.py:143-174 prep_im_for_blob + :898-923 im_list_to_blob on the device: uint8 [h,w,3] (BGR)
    -> fp32 blob [1,3,Hp,Wp] (mean-subtracted, bilinearly resized by `scale`, zero-padded to a multiple of `stride`)
    and the resized (h, w).  flip=True mirrors the image first (get_image_blob's im[:, ::-1, :] for a flipped roidb
    entry), bit-identical to passing a flipped copy.  out: a float32 CUDA buffer of at least 3*Hp*Wp elements whose
    leading part receives the blob (padding written as zeros); the blob returned is then a view of it."""
    require_cuda(image_hwc_u8)
    assert image_hwc_u8.dtype == torch.uint8 and image_hwc_u8.dim() == 3 and image_hwc_u8.shape[2] == 3
    im = image_hwc_u8.contiguous()
    h, w = int(im.shape[0]), int(im.shape[1])
    ho, wo = int(np.rint(h * scale)), int(np.rint(w * scale))              # cvRound(src * f) (cv2.resize dsize rule)
    Hp, Wp = int(math.ceil(ho / float(stride)) * stride), int(math.ceil(wo / float(stride)) * stride)
    if out is None:
        blob = torch.empty((1, 3, Hp, Wp), dtype=torch.float32, device=im.device)
    else:
        assert out.dtype == torch.float32 and out.is_contiguous() and out.device == im.device
        if out.numel() < 3 * Hp * Wp:
            raise ValueError("prep_image: out holds %d elements, the blob needs %d" % (out.numel(), 3 * Hp * Wp))
        blob = out.reshape(-1)[:3 * Hp * Wp].view(1, 3, Hp, Wp)
    pm = (C.c_double * 3)(*[float(v) for v in pixel_means])
    with _Timed("prep_image", 1, {"bytes": 3.0 * h * w + 12.0 * Hp * Wp}, im.device):
        call("prep_image", im.device, im, h, w, float(scale), ho, wo, Hp, Wp, pm, blob, int(bool(flip)))
    return blob, (ho, wo)


def label_restore_geometry(im_info):
    """(h, w, fx, out_h, out_w) of upsnet_end2end_test.py:259-266 for one im_info row [h, w, scale].  im_info is float32
    in the reference (coco.py:145-147), so fx = 1 / im_info[2] is a float32 that cv2 receives as a double, and the crop
    is int() of the float32 entries; the output size is cv2's cvRound(h * fx) (half to even)."""
    info = np.asarray(im_info, dtype=np.float32).reshape(-1)[:3]
    h, w = int(info[0]), int(info[1])
    fx = float(np.float32(1) / info[2])
    return h, w, fx, int(np.rint(h * fx)), int(np.rint(w * fx))


def label_restore_index(n_out, fx, n_crop):
    """Source indices of one axis of the restore (the rule upsnet_label_restore applies on the device): cv2's
    INTER_NEAREST min(floor(i * (1 / fx)), n_crop - 1) for i < n_out, with 1 / fx and the product in double."""
    return np.minimum(np.floor(np.arange(n_out, dtype=np.float64) * (1.0 / fx)).astype(np.int64), n_crop - 1)


def label_restore(label_map, im_info, *more_maps):
    """upsnet_end2end_test.py:259-266 on the device: crop an int64 label map [Hp,Wp] (or [1,Hp,Wp]) to im_info[:2],
    wrap it to uint8 like astype('uint8') and resize it back to the original image size with cv2's INTER_NEAREST rule.
    Returns int64 with the input's leading dimensions and [out_h,out_w] last, so it feeds unified_pan_result unchanged.
    A second map of the same shape may follow im_info: both are restored in one launch and a tuple is returned."""
    assert len(more_maps) <= 1, "label_restore takes one or two maps"
    maps = (label_map,) + tuple(more_maps)
    require_cuda(*maps)
    Hp, Wp = int(label_map.shape[-2]), int(label_map.shape[-1])
    lead = tuple(label_map.shape[:-2])
    srcs = []
    for m in maps:
        assert tuple(m.shape) == tuple(label_map.shape) and m.numel() == Hp * Wp, "one [Hp,Wp] map per call"
        srcs.append(m.reshape(Hp, Wp).to(torch.int64).contiguous())
    h, w, fx, oh, ow = label_restore_geometry(im_info)
    if not (0 < h <= Hp and 0 < w <= Wp):
        raise ValueError("im_info crop (%d, %d) outside the %dx%d label map" % (h, w, Hp, Wp))
    dev = srcs[0].device
    outs = [torch.empty(lead + (oh, ow), dtype=torch.int64, device=dev) for _ in srcs]
    two = len(srcs) == 2
    with _Timed("label_restore", 1, {"bytes": 16.0 * oh * ow * len(srcs)}, dev):
        call("label_restore", dev, srcs[0], srcs[1] if two else None, Hp, Wp, h, w, fx, oh, ow,
             outs[0], outs[1] if two else None)
    return tuple(outs) if two else outs[0]


# ------------------------------------------------------------------------------------------------
# Row f4: im_post (upsnet_end2end_test.py:95-152) -- mask paste + COCO RLE
# ------------------------------------------------------------------------------------------------
_impost_ws = _Workspace()


def rle_to_string(cnts):
    """pycocotools maskApi.c rleToString: the compressed `counts` bytes of a COCO RLE from its run lengths (host side; a
    pure function of the numbers the device kernel produces)."""
    out = bytearray()
    cnts = [int(c) for c in cnts]
    for i, x in enumerate(cnts):
        if i > 2:
            x -= cnts[i - 2]
        more = True
        while more:
            c = x & 0x1f
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            if more:
                c |= 0x20
            out.append(c + 48)
    return bytes(out)


def rle_from_string(s):
    """pycocotools maskApi.c rleFrString, the inverse of rle_to_string: uint32 run lengths from the compressed `counts`
    of a COCO RLE (str or bytes)."""
    if isinstance(s, str):
        s = s.encode()
    cnts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return np.asarray(cnts, np.int64).astype(np.uint32)


MAX_POLY_COORD = 4e8       # (int)(5 * c + .5) stays inside int32, as maskApi.c needs


# One image's segmentations in upsnet_gt_rle's layout (see pack_segmentations)
PackedSegms = collections.namedtuple("PackedSegms", "ann_poly poly_vert verts src_off src_counts bound sizes")


def pack_segmentations(segms, h, w):
    """COCO.annToRLE's inputs for upsnet_gt_rle, in annotation order.  A list segmentation is dispatched as
    maskUtils.frPyObjects does: len(segm[0]) == 4 reads every entry as a box [x, y, bw, bh] (rleFrBbox: the polygon
    [xs, ys, xs, ye, xe, ye, xe, ys], xe = xs + bw and ye = ys + bh in float64); len(segm[0]) > 4 makes every entry a
    polygon of k = len(p) // 2 vertices (later ones of 4 or 2 coordinates included); anything else, and an empty list,
    raises ValueError.  Polygons are rasterised at (h, w), the image record's size.  Any other segmentation (compressed
    or uncompressed RLE dict, [H,W] mask) is parsed by evaluation.gt_rle into host run lengths that the device copies
    through.  -> PackedSegms: ann_poly int32 [G+1], poly_vert int32 [P+1], verts float64 [V*2], src_off int64 [G+1],
    src_counts uint32, bound (int: the run capacity, see upsnet_gt_rle) and sizes int [2, G] (the RLE h, w)."""
    import itertools
    from .evaluation import gt_rle
    h, w = int(h), int(w)
    if h <= 0 or w <= 0:
        raise ValueError("image size %dx%d is empty" % (h, w))
    polys, ann_poly, src, src_len, sizes = [], [0], [], [], []
    for seg in segms:
        if isinstance(seg, list):
            if not seg:
                raise ValueError("an empty polygon list (pycocotools' frPyObjects indexes segm[0])")
            n0 = len(seg[0])
            if n0 == 4:
                bb = np.asarray(seg, np.float64)            # ragged rows raise, as frBbox's 2-D double buffer does
                if bb.ndim != 2 or bb.shape[1] != 4:
                    raise ValueError("a box-list segmentation must be [[x, y, w, h], ...]")
                xs, ys = bb[:, 0], bb[:, 1]
                xe, ye = xs + bb[:, 2], ys + bb[:, 3]
                polys.extend(np.stack([xs, ys, xs, ye, xe, ye, xe, ys], 1))
            elif n0 > 4:
                polys.extend(seg)
            else:
                raise ValueError("segmentation %r...: input type is not supported (frPyObjects)" % (seg[:1],))
            src_len.append(0)
            sizes.append((h, w))
        else:
            rh, rw, cnts = gt_rle(seg)
            src.append(cnts)
            src_len.append(cnts.size)
            sizes.append((rh, rw))
        ann_poly.append(len(polys))
    k = np.fromiter((len(p) // 2 for p in polys), np.int64, len(polys))
    poly_vert = np.zeros(len(polys) + 1, np.int64)
    np.cumsum(k, out=poly_vert[1:])
    verts = np.fromiter(itertools.chain.from_iterable(p[:2 * n] for p, n in zip(polys, k.tolist())), np.float64,
                        2 * int(poly_vert[-1]))
    if not np.all(np.abs(verts) < MAX_POLY_COORD):
        raise ValueError("polygon coordinates must be finite and below %g in magnitude" % MAX_POLY_COORD)
    ann_poly = np.asarray(ann_poly, np.int64)
    src_len = np.asarray(src_len, np.int64)
    # the run bound: 1 + per edge min(w, (|X1 - X0| + 1) // 5 + 1) over the annotation's polygons, at most h * w + 1
    X = np.trunc(5.0 * verts[0::2] + .5).astype(np.int64)
    nxt = np.arange(X.size) + 1
    full = k > 0
    nxt[poly_vert[1:][full] - 1] = poly_vert[:-1][full]
    per_edge = np.minimum(w, (np.abs(X[nxt] - X) + 1) // 5 + 1) if X.size else np.zeros(0, np.int64)
    ann_of_vert = np.repeat(np.repeat(np.arange(len(segms)), np.diff(ann_poly)), k)
    edges = np.bincount(ann_of_vert, weights=per_edge, minlength=len(segms)).astype(np.int64)
    is_poly = np.diff(ann_poly) > 0
    bound = int(np.where(is_poly, np.minimum(edges + 1, h * w + 1), src_len).sum())
    src_off = np.zeros(len(segms) + 1, np.int64)
    np.cumsum(src_len, out=src_off[1:])
    return PackedSegms(ann_poly=ann_poly.astype(np.int32), poly_vert=poly_vert.astype(np.int32), verts=verts,
                       src_off=src_off, src_counts=np.concatenate(src).astype(np.uint32) if src else np.zeros(0, np.uint32),
                       bound=bound, sizes=np.asarray(sizes, np.int64).reshape(-1, 2).T)


def gt_rle_arrays(pk):
    """The host arrays upsnet_gt_rle reads, in the order gt_rle_call takes their device addresses."""
    return [pk.verts, pk.src_off, pk.ann_poly, pk.poly_vert, pk.src_counts]


def gt_rle_call(pk, h, w, ptrs, counts, offsets, err, ws):
    """Launches upsnet_gt_rle on the current stream for a PackedSegms whose gt_rle_arrays() were staged at the device
    addresses ptrs; counts int32 [>= pk.bound], offsets int64 [G + 1], err device int32 [1], ws its workspace."""
    call("gt_rle", counts.device, int(h), int(w), len(pk.ann_poly) - 1, ptrs[2], ptrs[3], ptrs[0], ptrs[1], ptrs[4],
         counts, counts.numel(), offsets, err, ws, ws.numel())


def ann_to_rle(segms, h, w, device=None, err=None):
    """COCO.annToRLE of one image's segmentations on the device (upsnet_gt_rle), at the image record's (h, w): polygon
    lists and box lists (see pack_segmentations) are rasterised by maskApi.c's rleFrPoly rule and their parts united,
    RLE dicts (compressed or uncompressed) and [H,W] masks are copied through.  Returns (counts int32 [>= total] holding
    the uint32 run lengths back to back, offsets int64 [G+1]) on the device; annotation g's runs are
    counts[offsets[g]:offsets[g+1]].  err: optional device int32 [1] that gets UPSNET_GT_RLE_E_CAPACITY OR-ed in if the
    runs outgrow the host's bound (then every offset is 0).  Nothing waits for the device."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    pk = pack_segmentations(segms, h, w)
    G = len(pk.ann_poly) - 1
    arrays = gt_rle_arrays(pk)
    offs = np.cumsum([0] + [a.nbytes + (-a.nbytes) % 8 for a in arrays])
    host = torch.empty((max(int(offs[-1]), 8),), dtype=torch.uint8, pin_memory=True)
    for a, o in zip(arrays, offs):
        host.numpy()[o:o + a.nbytes] = a.view(np.uint8)
    stage = host.to(dev, non_blocking=True)
    out = (torch.empty((max(pk.bound, 1),), dtype=torch.int32, device=dev),
           torch.empty((G + 1,), dtype=torch.int64, device=dev))
    if err is None:
        err = torch.zeros((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((max(query_bytes("gt_rle_workspace_bytes", G, int(h), int(w)), 1),), dtype=torch.uint8, device=dev)
    gt_rle_call(pk, h, w, [C.c_void_p(stage.data_ptr() + int(o)) for o in offs[:-1]], out[0], out[1], err, ws)
    return out


def im_post_rle(pred_boxes, pred_masks, cls_inds, im_h, im_w, n_dev=None, cap=None):
    """upsnet_im_post_rle: the COCO run lengths of every detection's pasted mask, computed on the device without
    materialising the [H,W] images.  pred_boxes [n,4] or [n,5] (batch index first, like the model's `pred_boxes`),
    pred_masks [n,C,M,M] probabilities, cls_inds [n].  Returns (counts uint32 [n,cap] as int64-viewable tensor, run_len
    int32 [n]) on the device; raises if a detection needs more than `cap` counts (default 16 per image column)."""
    require_cuda(pred_boxes, pred_masks, cls_inds)
    boxes = f32c(pred_boxes[:, 1:] if pred_boxes.shape[1] == 5 else pred_boxes)
    masks = f32c(pred_masks)
    n, Cc, M, M2 = masks.shape
    assert M == M2 and boxes.shape == (n, 4) and cls_inds.numel() == n
    cls = cls_inds.to(torch.int64).contiguous()
    dev = masks.device
    cap = int(cap) if cap else 16 * int(im_w) + 64
    nb = query_bytes("im_post_workspace_bytes", n, cap)
    ws = _impost_ws.get(dev, nb)
    counts = torch.empty((max(n, 1), cap), dtype=torch.int32, device=dev)      # uint32 payload
    run_len = torch.zeros((max(n, 1),), dtype=torch.int32, device=dev)
    ovf = torch.zeros((1,), dtype=torch.int32, device=dev)
    with _Timed("im_post", 1, {"bytes": 4.0 * masks.numel()}, dev):
        call("im_post_rle", dev, masks, Cc, M, boxes, cls, n, n_dev, int(im_h), int(im_w), counts,
             cap, run_len, ovf, ws, ws.numel())
    return counts[:n], run_len[:n], ovf


def im_post(boxes_all, masks_all, scores, pred_boxes, pred_masks, cls_inds, num_classes, im_info):
    """Drop-in for upsnet_end2end_test.py:95-152 `im_post` (same arguments, same side effects on boxes_all / masks_all):
    device tensors in, per-class lists of [x1,y1,x2,y2,score] arrays and COCO RLE dicts out.  One kernel launch and one
    D2H copy of the run lengths per image instead of n x (cv2.resize + paste + pycocotools encode) on the host."""
    H, W = int(im_info[0]), int(im_info[1])
    counts, run_len, ovf = im_post_rle(pred_boxes, pred_masks, cls_inds, H, W)
    if int(ovf.item()):
        raise UpsnetError("im_post: a mask needs more RLE counts than the buffer holds (pass a larger cap)")
    rl = run_len.cpu().numpy()
    cn = counts.cpu().numpy().view(np.uint32)
    boxes_np = (pred_boxes[:, 1:] if pred_boxes.shape[1] == 5 else pred_boxes).float().cpu().numpy()
    sc = scores.float().cpu().numpy().reshape(-1, 1)
    ci = cls_inds.cpu().numpy()
    for idx in range(1, num_classes):
        sel = np.flatnonzero(ci == idx)
        cls_boxes = np.hstack([boxes_np[sel], sc[sel]]) if sel.size else np.zeros((0, 5), np.float32)
        segms = [{"size": [H, W], "counts": rle_to_string(cn[d, :rl[d]]).decode()} for d in sel]
        boxes_all[idx].append(cls_boxes)
        masks_all[idx].append(segms)


# ------------------------------------------------------------------------------------------------
# combined panoptic result (dataset/base_dataset.py:373-449): instance output merged with the semantic head
# ------------------------------------------------------------------------------------------------
_comb_ws = _Workspace()
COMBINED_ERRORS = ((1, "a detection needs more RLE counts than im_post_rle's buffer holds"),
                   (2, "an RLE whose runs do not cover the semantic map (mask size != semantic map size)"),
                   (4, "more than 2048 detections"))


def combined_pan_result(sem, scores, cls_inds, rle, num_seg_classes, num_classes, score_threshold=0.6,
                        fraction_threshold=0.7, stuff_area_limit=4 * 64 * 64, n_dev=None, check_errors=True):
    """dataset/base_dataset.py:373-449 get_combined_pan_result + _merge_pred_single_core for one image, on the device.
    sem int64 or uint8 [H,W] / [1,H,W] (the restored semantic map; int64 values wrap to uint8); scores fp32 [n] and
    cls_inds [n] of the detections (classes outside [1, num_classes) are ignored, as im_post drops them); rle = (counts,
    run_len) as im_post_rle returns them, of an H x W image; n_dev optional device count <= n.  Detections are taken by
    descending score, ties by the later position in im_post's class-ascending concatenation (class desc, index desc).
    -> uint8 [H,W,3] (class, instance number, 0).  Sync-free unless check_errors (one int D2H: raises ValueError for a
    mask size that differs from the map's, UpsnetError for the other error bits)."""
    counts, run_len = rle[0], rle[1]
    require_cuda(sem, scores, cls_inds, counts, run_len, n_dev)
    if sem.dtype not in (torch.uint8, torch.int64):
        sem = sem.to(torch.int64)
    sem = sem.reshape(sem.shape[-2:]).contiguous()
    H, W = int(sem.shape[0]), int(sem.shape[1])
    if H * W > 1 << 24:
        raise ValueError("combined_pan_result: %dx%d image: the reference's float32 pixel counts are exact up to 2^24 "
                         "pixels only" % (H, W))
    sc = f32c(scores.reshape(-1))
    cls = cls_inds.reshape(-1).to(torch.int64).contiguous()
    n = int(sc.numel())
    assert cls.numel() == n and run_len.numel() >= n and (n == 0 or counts.shape[0] >= n)
    cap = int(counts.shape[1]) if counts.dim() == 2 else 1
    cn, rl = counts.contiguous(), run_len.to(torch.int32).contiguous()
    dev = sem.device
    nb = query_bytes("combined_pan_workspace_bytes", n, H, W)
    ws = _comb_ws.get(dev, nb)
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
    err = torch.zeros((1,), dtype=torch.int32, device=dev)
    with _Timed("combined_pan", 3, {"bytes": (sem.element_size() * 2 + 3.25) * H * W}, dev):
        call("combined_pan_result", dev, sem, sem.element_size(), H, W, sc, cls, n, n_dev,
             cn, cap, rl, int(num_seg_classes), int(num_classes),
             float(score_threshold), float(fraction_threshold), int(stuff_area_limit),
             out, err, ws, ws.numel())
    if check_errors:
        e = int(err.item())
        if e & 2:
            raise ValueError("combined_pan_result: " + COMBINED_ERRORS[1][1])
        if e:
            raise _lib.UpsnetError("combined_pan_result: " + "; ".join(m for b, m in COMBINED_ERRORS if e & b))
    return out


def combined_inputs(boxes, masks, i, H, W):
    """Host side of get_combined_pan_result for image i: the per-class lists concatenated in ascending class order (the
    reference's order before its sort) -> scores fp32 [n], classes int64 [n], counts uint32 [max(n,1), cap] and run_len
    int32 [max(n,1)] in im_post_rle's layout.  Compressed `counts` strings are parsed with rle_from_string; lists of run
    lengths are taken as they are.  A mask whose size is not (H, W) raises ValueError (the reference fails to broadcast)."""
    sc, cl, runs = [], [], []
    for j in range(1, len(boxes)):
        b = np.asarray(boxes[j][i], np.float32).reshape(-1, 5)
        ms = masks[j][i]
        assert len(ms) == b.shape[0], "boxes[%d][%d] and masks[%d][%d] differ in length" % (j, i, j, i)
        for m in ms:
            if [int(v) for v in m["size"]] != [int(H), int(W)]:
                raise ValueError("mask size %s != semantic map size %s (image %d)" % (list(m["size"]), [H, W], i))
            c = m["counts"]
            runs.append(rle_from_string(c) if isinstance(c, (str, bytes)) else np.asarray(c, np.int64).astype(np.uint32))
        sc.append(b[:, 4])
        cl.append(np.full(b.shape[0], j, np.int64))
    n = len(runs)
    cap = max([r.size for r in runs] + [1])
    cn = np.zeros((max(n, 1), cap), np.uint32)
    rl = np.zeros(max(n, 1), np.int32)
    for d, r in enumerate(runs):
        cn[d, :r.size] = r
        rl[d] = r.size
    sc = np.concatenate(sc).astype(np.float32) if sc else np.zeros(0, np.float32)
    cl = np.concatenate(cl) if cl else np.zeros(0, np.int64)
    return sc, cl, cn, rl


def get_combined_pan_result(segs, boxes, masks, num_seg_classes, num_classes, score_threshold=0.6,
                            fraction_threshold=0.7, stuff_area_limit=4 * 64 * 64, device=None):
    """Drop-in for dataset/base_dataset.py:373-403 get_combined_pan_result on the test script's results (all_ssegs,
    all_boxes, all_masks): segs[i] uint8 [H,W]; boxes[j][i] [n_ij,5] (score in column 4) and masks[j][i] COCO RLE dicts
    for classes j = 1 .. len(boxes) - 1.  Each image's compressed strings are parsed on the host and uploaded once; the
    merge runs on the device.  -> list of uint8 [H,W,3] numpy maps.  The reference's num_seg_classes / num_classes come
    from config.dataset; here they are arguments.  `segs` is not modified."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = []
    for i, seg in enumerate(segs):
        seg = np.ascontiguousarray(seg)
        sc, cl, cn, rl = combined_inputs(boxes, masks, i, seg.shape[0], seg.shape[1])
        # one pinned upload of everything the image needs
        tensors = [torch.from_numpy(a) for a in (seg, sc, cl, cn.view(np.int32), rl)]
        seg_d, sc_d, cl_d, cn_d, rl_d = [t.pin_memory().to(dev, non_blocking=True) for t in tensors]
        pan = combined_pan_result(seg_d, sc_d, cl_d, (cn_d, rl_d), num_seg_classes, num_classes, score_threshold,
                                  fraction_threshold, stuff_area_limit)
        out.append(pan.cpu().numpy())
    return out
