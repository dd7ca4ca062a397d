"""Thin Python wrappers over the C ABI: the conv / stem descriptor builders, which take device addresses and shapes (no
GPU needed), and launch functions over torch CUDA tensors used purely as device memory.  All layout decisions (NHWC,
channel slices, bf16x3 planes) are made by the caller (`yolov6_b200.engine`).
"""
import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib
from ._lib import ACT_CODES, DT_BF16, DT_F16, DT_F32, DT_U8, ConvDesc, DwDesc, SeDesc, StemDesc

# Names of the yv6_conv_plan (10) / yv6_conv_plan_host (12) output words.  a_res = A stages * 100 + CTA pair * 10 + B resident.
PLAN_KEYS = ("BW", "BH", "BI", "BN", "KB", "stages", "grid", "tiles", "halo", "a_res", "smem", "threads")


@dataclass(eq=False)
class Launch:
    """One kernel launch of an engine: library entry point `fn` (a name) called as fn(handle, *args, stream), or a callable
    fn(stream).  Descriptor launches pass `desc` by reference."""
    kind: str
    fn: object
    args: tuple = ()
    desc: object = None

    def run(self, lib, h, sp):
        if isinstance(self.fn, str):
            _lib.check(getattr(lib, self.fn)(h, *self.args, sp))
        else:
            self.fn(sp)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def bias_buffer(cout, device):
    """Zeroed fp32 bias buffer of Cout rounded up to a multiple of 256 (the kernel reads 16 floats at a time)."""
    return torch.zeros((cout + 255) // 256 * 256, dtype=torch.float32, device=device)


def pad_bias(bias, cout):
    """fp32 bias padded with zeros to a multiple of 256 (see bias_buffer)."""
    out = bias_buffer(cout, bias.device)
    out[:cout] = bias.float()
    return out


def split3(t):
    """fp32 -> stacked bf16 planes [3, ...] with hi + mid + lo == t to ~2^-24 relative."""
    t = t.float()
    p0 = t.to(torch.bfloat16)
    r1 = t - p0.float()
    p1 = r1.to(torch.bfloat16)
    r2 = r1 - p1.float()
    p2 = r2.to(torch.bfloat16)
    return torch.stack([p0, p1, p2])


def pair_view_weights(w33):
    """[Cout, 3, 3, Cin] weights of a 3x3 stride-2 conv -> [Cout, 3, 2, 2*Cin] weights of the same conv on the column-pair view
    [N, H, W/2, 2*Cin] of its input (3x2 kernel, stride (2, 1), pad (1, 1)): tap 0 = input columns (2j-2 | 2j-1), of which only the
    odd one is under the 3x3 window; tap 1 = (2j | 2j+1).  See include/yv6.h `stride_w` / `pair_view`."""
    cout, _, _, cin = w33.shape
    wf = torch.zeros(cout, 3, 2, 2 * cin, dtype=w33.dtype, device=w33.device)
    wf[:, :, 0, cin:] = w33[:, :, 0]
    wf[:, :, 1, :cin] = w33[:, :, 1]
    wf[:, :, 1, cin:] = w33[:, :, 2]
    return wf


def conv_desc(x, x_shape, w, w_shape, y, y_strides, *, x_c_off=0, bias=0, stride=1, act=None, y_c_off=0, y_elem_off=0,
              y_f32=False, res=None, res_c_off=0, res_strides=None, alpha=1.0, accumulate=False, nsplit=1, pad=None, out_hw=None,
              stride_w=0, pair_view=0, force=None, f16=False):
    """yv6_conv_desc of y[..., y_c_off:+Cout] = act(conv(x[..., x_c_off:+Cin], w) + bias) (+ alpha * res), built from device
    addresses (ints) and shapes only, so that launches can be described and planned without a GPU.

    x: bf16 NHWC buffer of shape x_shape = (N, H, W, channel pitch); w: bf16 KRSC weights of shape w_shape = (Cout, kh, kw, Cin);
    bias: padded fp32 (pad_bias) or 0; y: bf16 (fp32 if y_f32) output whose element (n, ho, wo, c) is at
    y + y_elem_off + c + n * y_strides[0] + ho * y_strides[1] + wo * y_strides[2]; res: bf16 residual laid out the same way with
    res_strides, or accumulate = True: y += conv(...) (the residual epilogue reads the old value of the same element).
    nsplit = 3: x, w, res and a bf16 y are each three contiguous bf16 planes.  pad = (rows, columns), default kh // 2 for both.
    force: {"bw": 8, ...} -> the descriptor's force_* tuning overrides.  f16: x, w, res and a 16-bit y are fp16 instead of bf16
    (nsplit = 1)."""
    N, H, W, Ct = x_shape
    Cout, kh, kw, Cin = w_shape
    planes = nsplit == 3
    d = ConvDesc()
    d.x = x + x_c_off * 2
    d.N, d.H, d.W, d.Cin, d.x_c_total = N, H, W, Cin, Ct
    d.x_plane_stride = N * H * W * Ct if planes else 0
    d.w = w
    d.w_plane_stride = Cout * kh * kw * Cin if planes else 0
    d.bias = bias
    d.Cout, d.kh, d.kw, d.stride = Cout, kh, kw, stride
    d.pad, d.pad_w = (kh // 2, _lib.PAD_SAME) if pad is None else pad
    if out_hw is not None:
        d.out_h, d.out_w = out_hw
    d.stride_w, d.pair_view = stride_w, pair_view
    d.act = ACT_CODES[act]
    d.y = y + (y_c_off + y_elem_off) * (4 if y_f32 else 2)
    d.y_dtype = DT_F32 if y_f32 else DT_F16 if f16 else DT_BF16
    d.reserved0 = DT_F16 if f16 else 0
    d.y_img_stride, d.y_h_stride, d.y_w_stride = y_strides
    d.y_plane_stride = N * y_strides[0] if planes and not y_f32 else 0
    if accumulate:
        res, res_c_off, res_strides, alpha = d.y, 0, y_strides, 1.0
    if res is not None:
        d.res = res + res_c_off * 2
        d.res_img_stride, d.res_h_stride, d.res_w_stride = res_strides
        d.res_plane_stride = N * res_strides[0] if planes else 0
        d.alpha = alpha
    d.nsplit = nsplit
    for k, v in (force or {}).items():
        setattr(d, "force_" + k, int(v))
    return d


def plan_of(d, device=0):
    """Tile plan yv6_conv_fwd would use for descriptor d on a device: {PLAN_KEYS[i]: value}."""
    out = (C.c_int32 * 10)()
    _lib.check(_lib.lib().yv6_conv_plan(_lib.handle(device), C.byref(d), out))
    return dict(zip(PLAN_KEYS, out))


def stem_desc(x, N, H, W, u8, w, bias, cout, act, y, nsplit=1, y_plane_stride=0, fp32_math=0):
    """yv6_stem_desc from device addresses: x [N,3,H,W] fp32 (uint8 if u8, scaled by 1/255), w fp32 [3][3][3][Cout], bias fp32
    [Cout] or 0, y NHWC bf16 (nsplit planes y_plane_stride apart)."""
    d = StemDesc()
    d.x, d.x_dtype, d.in_scale = x, DT_U8 if u8 else DT_F32, 1.0 / 255.0
    d.N, d.H, d.W = N, H, W
    d.w, d.bias, d.Cout, d.act = w, bias, cout, ACT_CODES[act]
    d.y, d.y_plane_stride, d.nsplit, d.fp32_math = y, y_plane_stride, nsplit, fp32_math
    return d


def dw_desc(x, x_shape, x_plane, w, bias, C, k, stride, act, y, y_pitch, y_plane=0, nsplit=1):
    """yv6_dw_desc from device addresses: x / y point at the first channel of their slices; x_shape = (N, H, W, channel pitch);
    w fp32 [k*k][C], bias fp32 [C] or 0."""
    d = DwDesc()
    d.x, (d.N, d.H, d.W, d.x_c_total), d.C = x, x_shape, C
    d.y, d.y_c_total = y, y_pitch
    d.x_plane_stride, d.y_plane_stride = (x_plane, y_plane) if nsplit == 3 else (0, 0)
    d.w, d.bias, d.k, d.stride, d.act, d.nsplit = w, bias, k, stride, ACT_CODES[act], nsplit
    return d


def se_desc(x, N, HW, C, Cr, pitch, plane, w1, b1, w2, b2, nsplit=1, f16=False):
    """yv6_se_desc from device addresses: x is the first channel of the slice scaled in place (fp16 if f16)."""
    d = SeDesc()
    d.x, d.N, d.HW, d.C, d.Cr, d.c_total, d.plane_stride = x, N, HW, C, Cr, pitch, plane if nsplit == 3 else 0
    d.w1, d.b1, d.w2, d.b2, d.nsplit, d.reserved0 = w1, b1, w2, b2, nsplit, DT_F16 if f16 else 0
    return d


def dwconv_fwd(x, w, bias, y, *, k, stride=1, act=None, x_c_offset=0, y_c_offset=0, nsplit=1, stream=None):
    """y[..., y_c_offset:+C] = act(depthwise_conv(x[..., x_c_offset:+C], w) + bias).  x / y: [N,H,W,pitch] bf16 ([3,...] when
    nsplit=3) or fp16; w fp32 [k*k][C]; bias fp32 [C] or None."""
    planes = nsplit == 3
    xs, ys = (x.shape[1:], y.shape[1:]) if planes else (x.shape, y.shape)
    d = dw_desc(x.data_ptr() + 2 * x_c_offset, tuple(xs), x.stride(0) if planes else 0, w.data_ptr(),
                bias.data_ptr() if bias is not None else 0, w.shape[1], k, stride, act, y.data_ptr() + 2 * y_c_offset, ys[-1],
                y.stride(0) if planes else 0, nsplit)
    fn = _lib.lib().yv6_dwconv_fwd_f16 if x.dtype == torch.float16 else _lib.lib().yv6_dwconv_fwd
    _lib.check(fn(_lib.handle(x.device.index or 0), C.byref(d), _lib.stream_ptr(stream)))
    return y


def se_fwd(x, w1, b1, w2, b2, *, c_offset=0, nsplit=1, stream=None):
    """SEBlock in place on x[..., c_offset:+C] (x: [N,H,W,pitch] bf16 or fp16, [3,...] when nsplit=3); w1 [Cr, C], w2 [C, Cr] fp32."""
    planes = nsplit == 3
    N, H, W, pitch = x.shape[1:] if planes else x.shape
    d = se_desc(x.data_ptr() + 2 * c_offset, N, H * W, w1.shape[1], w1.shape[0], pitch, x.stride(0) if planes else 0,
                w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(), nsplit, x.dtype == torch.float16)
    _lib.check(_lib.lib().yv6_se_fwd(_lib.handle(x.device.index or 0), C.byref(d), _lib.stream_ptr(stream)))
    return x


def conv_fwd(x, w, bias, y, *, cin=None, x_c_offset=0, stride=1, act=None, y_c_offset=0,
             y_img_stride=None, y_h_stride=None, y_w_stride=None, y_elem_offset=0,
             res=None, res_c_offset=0, alpha=1.0, nsplit=1, force=None, stream=None, pad=None, out_hw=None, stride_w=0, pair_view=0):
    """y[..., y_c_offset:+Cout] = act(conv(x[..., x_c_offset:+Cin], w) + bias) (+ alpha*res).

    x: [N,H,W,Ct] bf16 (nsplit=1) or [3,N,H,W,Ct] (nsplit=3); w: [Cout,kh,kw,Cin] bf16 (or [3,...]);
    bias: padded fp32 (see pad_bias) or None; y: NHWC buffer, bf16 ([3,...] when nsplit=3) or fp32.  fp16 x, w, res and y (or
    fp32 y) select the fp16 operands.
    """
    planes = nsplit == 3
    ws = w.shape[1:] if planes else w.shape
    assert cin is None or cin == ws[3], (cin, ws[3])
    y_f32 = y.dtype == torch.float32
    yst = y.stride()[1:] if planes and not y_f32 else y.stride()
    y_strides = [s if o is None else o for s, o in zip(yst, (y_img_stride, y_h_stride, y_w_stride))]
    rst = None if res is None else (res.stride()[1:] if planes else res.stride())[:3]
    d = conv_desc(x.data_ptr(), x.shape[1:] if planes else x.shape, w.data_ptr(), ws, y.data_ptr(), y_strides, x_c_off=x_c_offset,
                  bias=bias.data_ptr() if bias is not None else 0, stride=stride, act=act, y_c_off=y_c_offset, y_elem_off=y_elem_offset,
                  y_f32=y_f32, res=None if res is None else res.data_ptr(), res_c_off=res_c_offset, res_strides=rst, alpha=alpha,
                  nsplit=nsplit, pad=pad, out_hw=out_hw, stride_w=stride_w, pair_view=pair_view, force=force, f16=x.dtype == torch.float16)
    dev = x.device.index or 0
    _lib.check(_lib.lib().yv6_conv_fwd(_lib.handle(dev), C.byref(d), _lib.stream_ptr(stream)))
    return y


def conv_plan(x_shape, w_shape, stride=1, nsplit=1, force=None, device=0, stride_w=0, pad=None, out_hw=None, pair_view=0, f16=False):
    """Tile plan (PLAN_KEYS) the kernel would use for a shape."""
    # plan only: non-null, aligned addresses
    d = conv_desc(16, x_shape, 16, w_shape, 16, (0, 0, 0), stride=stride, nsplit=nsplit, pad=pad, out_hw=out_hw, stride_w=stride_w,
                  pair_view=pair_view, force=force, f16=f16)
    return plan_of(d, device)
