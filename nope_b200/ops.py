"""Per-op entry points of the C ABI (include/nope_b200.h, "per-op entry points"), bound
for the parity tests: each runs ONE layer type of the reference UNet on fp32 NCHW CUDA
tensors through the same kernels the sweep uses."""
import ctypes as C

import torch

from . import _lib

_IMPL = {"tcgen05": 0, "simt": 1, "tcgen05_2cta": 2}


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(t):
    return None if t is None else t.to(torch.float32).contiguous()


def conv(x0, weight, bias=None, x1=None, mode="3x3", impl="tcgen05"):
    """mode '3x3' (pad 1), '1x1', 'unshuffle' (pixel-unshuffle(2) + 1x1; weight
    [Cout, 4*Cin, 1, 1]) or 'upsample3x3' (nearest x2 + conv3x3, folded into four 2x2 parity
    kernels; x0 is the low-resolution input).  x1 is concatenated after x0 along channels."""
    lib = _lib.load()
    m = {"3x3": 0, "1x1": 1, "unshuffle": 2, "upsample3x3": 3}[mode]
    x0, x1, weight, bias = _f32(x0), _f32(x1), _f32(weight), _f32(bias)
    n, c0, hin, win = x0.shape
    h, w = (hin // 2, win // 2) if m == 2 else ((2 * hin, 2 * win) if m == 3 else (hin, win))
    cout = weight.shape[0]
    out = torch.empty((n, cout, h, w), device=x0.device, dtype=torch.float32)
    with torch.cuda.device(x0.device):
        _lib.check(lib.nope_op_conv(_IMPL[impl], m, _lib.ptr(x0), c0, _lib.ptr(x1),
                                    0 if x1 is None else x1.shape[1], _lib.ptr(weight),
                                    _lib.ptr(bias), _lib.ptr(out), n, h, w, cout, _stream(x0.device)))
    return out


def conv_gn(x0, weight, bias, gamma, beta, groups, silu=True, x1=None, mode="3x3", impl="tcgen05"):
    """[SiLU](GroupNorm(conv(x))) with statistics from the conv epilogue (the sweep's path)."""
    lib = _lib.load()
    m = {"3x3": 0, "1x1": 1, "unshuffle": 2}[mode]
    x0, x1, weight, bias, gamma, beta = map(_f32, (x0, x1, weight, bias, gamma, beta))
    n, c0, hin, win = x0.shape
    h, w = (hin // 2, win // 2) if m == 2 else (hin, win)
    cout = weight.shape[0]
    out = torch.empty((n, cout, h, w), device=x0.device, dtype=torch.float32)
    with torch.cuda.device(x0.device):
        _lib.check(lib.nope_op_conv_gn(_IMPL[impl], m, _lib.ptr(x0), c0, _lib.ptr(x1),
                                       0 if x1 is None else x1.shape[1], _lib.ptr(weight),
                                       _lib.ptr(bias), _lib.ptr(gamma), _lib.ptr(beta), groups,
                                       1 if silu else 0, _lib.ptr(out), n, h, w, cout,
                                       _stream(x0.device)))
    return out


def conv_gn_fused(x0, weight, bias, gamma=None, beta=None, groups=8, silu=True, x1=None, mode="3x3",
                  precision=0, chan_bias=None, residual=None, res_div=0, want_emit=False):
    """The sweep's fused layer on the CTA-pair kernel: [SiLU](GroupNorm(conv(x))) + chan_bias +
    residual with everything after the convolution in its epilogue (groups=0: no normalisation).
    precision 0 fp16 / 1 exact weights / 2 split (hi + lo operands).  -> out [, emit [n, 2]]."""
    lib = _lib.load()
    m = {"3x3": 0, "1x1": 1, "unshuffle": 2}[mode]
    x0, x1, weight, bias, gamma, beta, chan_bias, residual = map(
        _f32, (x0, x1, weight, bias, gamma, beta, chan_bias, residual))
    n, c0, hin, win = x0.shape
    h, w = (hin // 2, win // 2) if m == 2 else (hin, win)
    cout = weight.shape[0]
    out = torch.empty((n, cout, h, w), device=x0.device, dtype=torch.float32)
    emit = torch.empty((n, 2), device=x0.device, dtype=torch.float32) if want_emit else None
    with torch.cuda.device(x0.device):
        _lib.check(lib.nope_op_conv_gn_fused(
            m, precision, _lib.ptr(x0), c0, _lib.ptr(x1), 0 if x1 is None else x1.shape[1],
            _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(gamma), _lib.ptr(beta), groups, 1 if silu else 0,
            _lib.ptr(chan_bias), _lib.ptr(residual), res_div, _lib.ptr(out), _lib.ptr(emit), n, h, w, cout,
            _stream(x0.device)))
    return (out, emit) if want_emit else out


def groupnorm(x, gamma, beta, groups, silu=False, chan_bias=None, residual=None):
    lib = _lib.load()
    x, gamma, beta = _f32(x), _f32(gamma), _f32(beta)
    chan_bias, residual = _f32(chan_bias), _f32(residual)
    n, c, h, w = x.shape
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _lib.check(lib.nope_op_groupnorm(_lib.ptr(x), _lib.ptr(gamma), _lib.ptr(beta), groups,
                                         1 if silu else 0, _lib.ptr(chan_bias), _lib.ptr(residual),
                                         _lib.ptr(out), n, c, h, w, _stream(x.device)))
    return out


def linear_attention(qkv, impl="simt"):
    """impl 'tcgen05' (both contractions on wgmma tensor cores; H*W a multiple of 128) or 'simt'."""
    lib = _lib.load()
    qkv = _f32(qkv)
    n, c, h, w = qkv.shape
    assert c == 384
    out = torch.empty((n, 128, h, w), device=qkv.device, dtype=torch.float32)
    with torch.cuda.device(qkv.device):
        _lib.check(lib.nope_op_linear_attention({"tcgen05": 0, "simt": 1}[impl], _lib.ptr(qkv), _lib.ptr(out),
                                                n, h, w, _stream(qkv.device)))
    return out


def attention(qkv):
    lib = _lib.load()
    qkv = _f32(qkv)
    n, c, h, w = qkv.shape
    assert c == 384
    out = torch.empty((n, 128, h, w), device=qkv.device, dtype=torch.float32)
    with torch.cuda.device(qkv.device):
        _lib.check(lib.nope_op_attention(_lib.ptr(qkv), _lib.ptr(out), n, h, w, _stream(qkv.device)))
    return out


def upsample2x(x):
    lib = _lib.load()
    x = _f32(x)
    n, c, h, w = x.shape
    out = torch.empty((n, c, 2 * h, 2 * w), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(lib.nope_op_upsample2x(_lib.ptr(x), _lib.ptr(out), n, c, h, w, _stream(x.device)))
    return out
