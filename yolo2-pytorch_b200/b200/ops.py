"""Tensor-level wrappers of the C ABI: each function checks device/dtype/contiguity, passes raw
device pointers plus torch's current CUDA stream, and raises RuntimeError on a non-zero code.
PyTorch is plumbing here (storage + streams); all arithmetic happens in libyolo2_b200.so."""
import ctypes

import torch

from . import lib as _l

OUT_F16_NHWC, OUT_F32_NCHW = 0, 1
CONV_A_TILED, CONV_WIDE_N = 1, 2
CONV_NO_STREAMK, CONV_FORCE_STREAMK, CONV_NO_SMALLK, CONV_PLAIN_STORE = 8, 1 << 30, 1 << 28, 1 << 29
CONV_POOL2X2, CONV_C32_IM2COL, CONV_C32_SWAP, CONV_CHAIN1X1 = 16, 32, 64, 128
FILTER_THRESHOLD, FILTER_FIX, FILTER_NONE = 0, 1, 2


launch_count = 0  # kernels of libyolo2_b200.so launched through this module (bench.py reports it)


def _ck(rc, what):
    global launch_count
    _l.check(rc, what)
    launch_count += 1


def conv_force_bn(bn):
    return bn << 8


def conv_force_mt(mt):
    return mt << 20


def conv_force_pair(v):
    """0 = auto, 1 = single-CTA tiles (the only form on sm_90; 2, CTA pairs, is rejected)."""
    return v << 22


CONV_ALLOW_PAIR = 4


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _req(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError('%s must be a CUDA tensor: the GPU path has no CPU fallback' % name)
    if t.dtype != dtype:
        raise TypeError('%s must be %s, got %s' % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError('%s must be contiguous' % name)
    return t


def pack_weight_f16(w, mode=0):
    """[Cout,Cin,k,k] fp32 -> fp16 [Cout,k,k,Cin] (mode 0) or [Cin,k,k,Cout] rotated (mode 1)."""
    _req(w, torch.float32, 'weight')
    cout, cin, k, _ = w.shape
    shape = (cout, k, k, cin) if mode == 0 else (cin, k, k, cout)
    out = torch.empty(shape, dtype=torch.float16, device=w.device)
    _ck(_l.load().yb_pack_weight_f16(_p(w), _p(out), cout, cin, k, mode, _s()), 'yb_pack_weight_f16')
    return out


SPLIT_SEGMENTS = {(True, False): (2, 0b00), (False, True): (2, 0b10), (True, True): (3, 0b100)}


def pack_weight_split_f16(w, split_a, split_w):
    """[Cout,Cin,k,k] fp32 -> fp16 [Cout,k,k,S*Cin], the concatenated B operand of the split-precision conv: segments
    [w_hi | w_hi] (activation split), [w_hi | w_lo] (weight split) or [w_hi | w_hi | w_lo] (both)."""
    _req(w, torch.float32, 'weight')
    cout, cin, k, _ = w.shape
    segments, lo_mask = SPLIT_SEGMENTS[(bool(split_a), bool(split_w))]
    out = torch.empty(cout, k, k, segments * cin, dtype=torch.float16, device=w.device)
    _ck(_l.load().yb_pack_weight_split_f16(_p(w), _p(out), cout, cin, k, segments, lo_mask, _s()), 'yb_pack_weight_split_f16')
    return out


def bn_fold(gamma, beta, mean, var, eps=1e-5):
    for n, t in (('gamma', gamma), ('beta', beta), ('mean', mean), ('var', var)):
        _req(t, torch.float32, n)
    c = gamma.numel()
    scale = torch.empty(c, dtype=torch.float32, device=gamma.device)
    shift = torch.empty_like(scale)
    _ck(_l.load().yb_bn_fold(_p(gamma), _p(beta), _p(mean), _p(var), float(eps), _p(scale), _p(shift), c, _s()), 'yb_bn_fold')
    return scale, shift


def _image(x, lut):
    """The first-layer input's (b, c, h, w) and the pointer arguments that carry it: fp32 NCHW [B,3,H,W], or with a table (the `_lut`
    entries) uint8 NHWC [B,H,W,3] and lut fp32 [3,256]."""
    if lut is None:
        _req(x, torch.float32, 'x')
        return tuple(x.shape), (_p(x),)
    _req(x, torch.uint8, 'x'); _req(lut, torch.float32, 'lut')
    if tuple(lut.shape) != (3, 256):
        raise ValueError('lut must be [3, 256], got %s' % (tuple(lut.shape),))
    b, h, wd, c = x.shape
    return (b, c, h, wd), (_p(x), _p(lut))


def conv0_bn_leaky_pool(x, w, scale, shift, slope, out=None, lut=None):
    """x fp32 NCHW [B,3,H,W] -> fp16 NHWC [B,H/2,W/2,32].  With `lut` (fp32 [3,256]): x uint8 NHWC [B,H,W,3] read through the table
    (yb_conv0_bn_leaky_pool_lut_fwd)."""
    _req(w, torch.float32, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    (b, c, h, wd), xa = _image(x, lut)
    if c != 3:
        raise ValueError('conv0 expects 3 input channels')
    cout = w.shape[0]
    if out is None:
        out = torch.empty(b, h // 2, wd // 2, cout, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    name = 'yb_conv0_bn_leaky_pool_fwd' if lut is None else 'yb_conv0_bn_leaky_pool_lut_fwd'
    _ck(getattr(_l.load(), name)(*xa, _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, cout, _s()), name)
    return out


def conv0_u8_bn_leaky_pool(x, w, scale, shift, slope, out=None):
    """x uint8 NHWC [B,H,W,3] (raw RGB frames; the kernel applies ToTensor's 1/255) -> fp16 NHWC [B,H/2,W/2,32]."""
    _req(x, torch.uint8, 'x'); _req(w, torch.float32, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    b, h, wd, c = x.shape
    if c != 3:
        raise ValueError('conv0 expects 3 input channels')
    cout = w.shape[0]
    if out is None:
        out = torch.empty(b, h // 2, wd // 2, cout, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_conv0_u8_bn_leaky_pool_fwd(_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, cout, _s()),
        'yb_conv0_u8_bn_leaky_pool_fwd')
    return out


def conv0_c64_bn_act(x, w, scale, shift, slope, pool=False, out=None, lut=None):
    """Conv2d(3, 64, 3, padding 1) + scale/shift + activation (+ 2x2 max-pool) of VGG's features.0 (yb_conv0_c64_bn_act_fwd):
    x fp32 NCHW [B,3,H,W], w fp32 [64,3,3,3], scale / shift fp32 [64] -> fp16 NHWC [B,H,W,64], or [B,H/2,W/2,64] with `pool`.
    With `lut` (fp32 [3,256]): x uint8 NHWC [B,H,W,3] read through the table (yb_conv0_c64_bn_act_lut_fwd)."""
    _req(w, torch.float32, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    (b, c, h, wd), xa = _image(x, lut)
    if c != 3 or tuple(w.shape) != (64, 3, 3, 3) or scale.numel() != 64 or shift.numel() != 64:
        raise ValueError('conv0_c64: x [B,3,H,W], w [64,3,3,3] and 64 scales / shifts expected')
    oh, ow = (h // 2, wd // 2) if pool else (h, wd)
    if out is None:
        out = torch.empty(b, oh, ow, 64, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    if tuple(out.shape) != (b, oh, ow, 64):
        raise ValueError('conv0_c64: out must be [%d,%d,%d,64]' % (b, oh, ow))
    name = 'yb_conv0_c64_bn_act_fwd' if lut is None else 'yb_conv0_c64_bn_act_lut_fwd'
    _ck(getattr(_l.load(), name)(*xa, _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, int(bool(pool)), _s()), name)
    return out


def _conv_common(fn_name, x, w, scale, shift, slope, out, batch, height, width, cin, cout, k, x_ld, y_ld, y_ch_off, out_mode, flags,
                 workspace=None):
    if workspace is not None and fn_name == 'yb_conv_bn_act_fwd':
        fn_name = 'yb_conv_bn_act_fwd_ws'
    fn = getattr(_l.load(), fn_name)
    args = [_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(out), batch, height, width, cin, cout, k, x_ld, y_ld, y_ch_off, out_mode]
    if fn_name != 'yb_conv_ref_fwd':
        args.append(flags)
    if fn_name == 'yb_conv_bn_act_fwd_ws':
        _req(workspace, torch.uint8, 'workspace')
        args += [_p(workspace), workspace.numel()]
    args.append(_s())
    _ck(fn(*args), fn_name)


def conv_workspace(device='cuda'):
    """Scratch buffer for stream-K convs (yb_conv_bn_act_fwd_ws): zero-filled once, one per stream / activation plan."""
    return torch.zeros(int(_l.load().yb_conv_workspace_bytes()), dtype=torch.uint8, device=device)


CONV_KERNELS = ('conv_igemm_kernel', 'conv_wide_kernel', 'conv_c32_kernel')


def conv_choice(batch, height, width, cin, cout, k, out_mode=OUT_F16_NHWC, flags=0, workspace=True):
    """The kernel and tile shape conv_bn_act picks for this shape (the library's own selection, yb_conv_choice).  `pooled`: the launch
    applies the fused 2x2 max-pool (CONV_POOL2X2; the library refuses the flag where it has no pooled form).  `chained`: the launch runs
    the following 1x1 unit in its epilogue (CONV_CHAIN1X1, conv_bn_act's `chain`; refused where this conv cannot be its producer)."""
    out = (ctypes.c_int * 6)()
    _l.check(_l.load().yb_conv_choice(batch, height, width, cin, cout, k, out_mode, flags, int(bool(workspace)), ctypes.byref(out)),
             'yb_conv_choice')
    return dict(kernel=CONV_KERNELS[out[0]], bk=out[1], bn=out[2], rows=out[3], streamk=bool(out[4]), grid=out[5],
                pooled=bool(flags & CONV_POOL2X2), chained=bool(flags & CONV_CHAIN1X1))


def conv_bn_act(x, w, scale, shift, slope, out=None, out_mode=OUT_F16_NHWC, y_ch_off=0, cin=None, flags=0, ref=False, workspace=None,
                chain=None):
    """x: fp16 [B,H,W,x_ld] (uses the first `cin` channels, default all); w: fp16 [Cout,k,k,Cin].
    out (fp16): [B,H,W,y_ld] written at channels [y_ch_off, y_ch_off+Cout); out (fp32): [B,Cout,H,W].
    flags & CONV_POOL2X2: the 2x2 max-pool is fused, out is [B,H/2,W/2,y_ld].
    chain = (w2, scale2, shift2, slope2): the 1x1 unit that reads this conv's output runs in the same launch (yb_conv_bn_act_chain_fwd),
    w2 fp16 [Cout2,1,1,Cout]; out is that unit's fp16 output [B,H,W,y_ld] at channels [y_ch_off, y_ch_off+Cout2)."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    b, h, wd, x_ld = x.shape
    cout, k, _, wcin = w.shape
    cin = wcin if cin is None else cin
    if cin != wcin:
        raise ValueError('weight Cin %d != %d' % (wcin, cin))
    if chain is not None:
        return _conv_chain(x, w, scale, shift, slope, chain, out, out_mode, y_ch_off, cin, flags, ref, workspace)
    if out is None:
        oh, ow = (h // 2, wd // 2) if (flags & CONV_POOL2X2) else (h, wd)
        out = (torch.empty(b, oh, ow, cout, dtype=torch.float16, device=x.device) if out_mode == OUT_F16_NHWC
               else torch.empty(b, cout, h, wd, dtype=torch.float32, device=x.device))
    if out_mode == OUT_F16_NHWC:
        _req(out, torch.float16, 'out')
        y_ld = out.shape[-1]
    else:
        _req(out, torch.float32, 'out')
        y_ld = 0
    if flags & CONV_POOL2X2:
        if ref:
            raise ValueError('conv_bn_act: the CUDA-core reference has no fused max-pool')
        if out.dim() != 4 or tuple(out.shape[:3]) != (b, h // 2, wd // 2) or y_ch_off < 0 or y_ch_off + cout > y_ld:
            raise ValueError('conv_bn_act: pooled out must be [%d,%d,%d,y_ld] with y_ch_off + Cout <= y_ld, got %s at y_ch_off %d'
                             % (b, h // 2, wd // 2, tuple(out.shape), y_ch_off))
    _conv_common('yb_conv_ref_fwd' if ref else 'yb_conv_bn_act_fwd', x, w, scale, shift, slope, out, b, h, wd, cin, cout, k, x_ld, y_ld,
                 y_ch_off, out_mode, flags, workspace=None if ref else workspace)
    return out


def round_up(n, m):
    return (n + m - 1) // m * m


def conv_bn_act_tail(x, w, scale, shift, slope, cin, out=None, out_mode=OUT_F16_NHWC, y_ch_off=0, flags=0):
    """yb_conv_bn_act_tail_fwd: conv_bn_act on the first `cin` channels of x (cin % 8 == 0, not necessarily of 32).
    x: fp16 [B,H,W,x_ld], x_ld >= cin; w: fp16 [Cout,k,k,round_up(cin, 32)], zero in channels >= cin (pack_weight_f16 of a weight
    zero-padded on Cin).  out as conv_bn_act."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    b, h, wd, x_ld = x.shape
    cout, k, _, cin_pad = w.shape
    if out is None:
        out = (torch.empty(b, h, wd, cout, dtype=torch.float16, device=x.device) if out_mode == OUT_F16_NHWC
               else torch.empty(b, cout, h, wd, dtype=torch.float32, device=x.device))
    if out_mode == OUT_F16_NHWC:
        _req(out, torch.float16, 'out')
        y_ld = out.shape[-1]
    else:
        _req(out, torch.float32, 'out')
        y_ld = 0
    _ck(_l.load().yb_conv_bn_act_tail_fwd(_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, cin, cin_pad, cout, k, x_ld, y_ld,
                                          y_ch_off, out_mode, flags, _s()), 'yb_conv_bn_act_tail_fwd')
    return out


def _conv_chain(x, w, scale, shift, slope, chain, out, out_mode, y_ch_off, cin, flags, ref, workspace):
    w2, scale2, shift2, slope2 = chain
    _req(w2, torch.float16, 'w2'); _req(scale2, torch.float32, 'scale2'); _req(shift2, torch.float32, 'shift2')
    b, h, wd, x_ld = x.shape
    cout, k = w.shape[0], w.shape[1]
    cout2 = w2.shape[0]
    if tuple(w2.shape) != (cout2, 1, 1, cout) or scale2.numel() != cout2 or shift2.numel() != cout2:
        raise ValueError('conv_bn_act chain: w2 must be [Cout2,1,1,%d] with Cout2 scales / shifts, got %s' % (cout, tuple(w2.shape)))
    if ref or out_mode != OUT_F16_NHWC:
        raise ValueError('conv_bn_act chain: the fused form has fp16 NHWC output and no CUDA-core reference')
    if out is None:
        out = torch.empty(b, h, wd, cout2, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    if out.dim() != 4 or tuple(out.shape[:3]) != (b, h, wd) or y_ch_off < 0 or y_ch_off + cout2 > out.shape[-1]:
        raise ValueError('conv_bn_act chain: out must be [%d,%d,%d,y_ld] with y_ch_off + Cout2 <= y_ld, got %s at y_ch_off %d'
                         % (b, h, wd, tuple(out.shape), y_ch_off))
    if workspace is not None:
        _req(workspace, torch.uint8, 'workspace')
    _ck(_l.load().yb_conv_bn_act_chain_fwd(_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(w2), _p(scale2), _p(shift2), float(slope2),
                                           _p(out), b, h, wd, cin, cout, cout2, k, x_ld, out.shape[-1], y_ch_off, flags, _p(workspace),
                                           0 if workspace is None else workspace.numel(), _s()), 'yb_conv_bn_act_chain_fwd')
    return out


def conv2d_out_size(size, k, stride, pad):
    return (size + 2 * pad - k) // stride + 1


def conv2d_choice(batch, height, width, cin, cout, kh, kw, stride=1, pad=(0, 0), out_mode=OUT_F16_NHWC, flags=0, workspace=True):
    """conv_choice for the general geometry (yb_conv2d_choice); height / width are the input dims, pad = (pad_h, pad_w)."""
    out = (ctypes.c_int * 6)()
    _l.check(_l.load().yb_conv2d_choice(batch, height, width, cin, cout, kh, kw, stride, pad[0], pad[1], out_mode, flags, int(bool(workspace)),
                                        ctypes.byref(out)), 'yb_conv2d_choice')
    return dict(kernel=CONV_KERNELS[out[0]], bk=out[1], bn=out[2], rows=out[3], streamk=bool(out[4]), grid=out[5],
                pooled=bool(flags & CONV_POOL2X2), chained=bool(flags & CONV_CHAIN1X1))


def conv2d_bn_act(x, w, scale, shift, slope, stride=1, pad=(0, 0), out=None, out_mode=OUT_F16_NHWC, y_ch_off=0, cin=None, flags=0, workspace=None):
    """yb_conv2d_bn_act_fwd: the conv_bn_act unit with kh x kw filters, stride 1 or 2 and zero padding pad = (pad_h, pad_w).
    x: fp16 [B,H,W,x_ld] (the first `cin` channels, default the weight's); w: fp16 [Cout,kh,kw,Cin] (pack_weight_khw_f16);
    out (fp16): [B,OH,OW,y_ld] written at channels [y_ch_off, y_ch_off+Cout); out (fp32): [B,Cout,OH,OW]."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    b, h, wd, x_ld = x.shape
    cout, kh, kw, wcin = w.shape
    cin = wcin if cin is None else cin
    if cin != wcin:
        raise ValueError('weight Cin %d != %d' % (wcin, cin))
    oh, ow = conv2d_out_size(h, kh, stride, pad[0]), conv2d_out_size(wd, kw, stride, pad[1])
    if out is None:
        out = (torch.empty(b, oh, ow, cout, dtype=torch.float16, device=x.device) if out_mode == OUT_F16_NHWC
               else torch.empty(b, cout, oh, ow, dtype=torch.float32, device=x.device))
    if out_mode == OUT_F16_NHWC:
        _req(out, torch.float16, 'out')
        y_ld = out.shape[-1]
    else:
        _req(out, torch.float32, 'out')
        y_ld = 0
    ws_ptr, ws_bytes = (None, 0) if workspace is None else (_p(_req(workspace, torch.uint8, 'workspace')), workspace.numel())
    _ck(_l.load().yb_conv2d_bn_act_fwd(_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, cin, cout, kh, kw, stride, pad[0], pad[1],
                                       x_ld, y_ld, y_ch_off, out_mode, flags, ws_ptr, ws_bytes, _s()), 'yb_conv2d_bn_act_fwd')
    return out


def pack_weight_khw_f16(w, cout_pad=None, cin_pad=None):
    """[Cout,Cin,kh,kw] fp32 -> fp16 [cout_pad,kh,kw,cin_pad], zero in the padded filters and channels."""
    _req(w, torch.float32, 'weight')
    cout, cin, kh, kw = w.shape
    cout_pad = cout if cout_pad is None else cout_pad
    cin_pad = cin if cin_pad is None else cin_pad
    out = torch.empty(cout_pad, kh, kw, cin_pad, dtype=torch.float16, device=w.device)
    _ck(_l.load().yb_pack_weight_khw_f16(_p(w), _p(out), cout, cin, kh, kw, cout_pad, cin_pad, _s()), 'yb_pack_weight_khw_f16')
    return out


def stem3x3_s2(x, w, scale, shift, pad=0, lut=None):
    """nn.Conv2d(3, 32, 3, stride 2, pad) + folded BatchNorm + ReLU: x fp32 NCHW [B,3,H,W] -> fp16 NHWC [B,OH,OW,32].  With `lut` (fp32
    [3,256]): x uint8 NHWC [B,H,W,3] read through the table (yb_stem3x3_s2_bn_relu_lut_fwd)."""
    _req(w, torch.float32, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    (b, c, h, wd), xa = _image(x, lut)
    if c != 3 or tuple(w.shape) != (32, 3, 3, 3):
        raise ValueError('stem3x3_s2: x [B,3,H,W] and w [32,3,3,3] expected')
    out = torch.empty(b, conv2d_out_size(h, 3, 2, pad), conv2d_out_size(wd, 3, 2, pad), 32, dtype=torch.float16, device=x.device)
    name = 'yb_stem3x3_s2_bn_relu_fwd' if lut is None else 'yb_stem3x3_s2_bn_relu_lut_fwd'
    _ck(getattr(_l.load(), name)(*xa, _p(w), _p(scale), _p(shift), _p(out), b, h, wd, pad, _s()), name)
    return out


def maxpool3x3_s2_valid(x, out=None, y_ch_off=0):
    """F.max_pool2d(x, 3, stride=2) on fp16 NHWC x [B,H,W,C] into channels [y_ch_off, y_ch_off + C) of out [B,OH,OW,y_ld]."""
    _req(x, torch.float16, 'x')
    b, h, w, c = x.shape
    if out is None:
        out = torch.empty(b, conv2d_out_size(h, 3, 2, 0), conv2d_out_size(w, 3, 2, 0), c, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_maxpool3x3_s2_valid_f16(_p(x), _p(out), out.shape[-1], y_ch_off, b, h, w, c, _s()), 'yb_maxpool3x3_s2_valid_f16')
    return out


def avgpool3x3_s1(x, out=None):
    """F.avg_pool2d(x, 3, stride=1, padding=1) (count_include_pad=True) on fp16 NHWC x [B,H,W,C]."""
    _req(x, torch.float16, 'x')
    b, h, w, c = x.shape
    out = torch.empty_like(x) if out is None else out
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_avgpool3x3_s1_f16(_p(x), _p(out), b, h, w, c, _s()), 'yb_avgpool3x3_s1_f16')
    return out


def avgpool3x3_s1_excl(x, out=None):
    """nn.AvgPool2d(3, stride=1, padding=1, count_include_pad=False) on fp16 NHWC x [B,H,W,C]: the divisor is the number of in-range pixels."""
    _req(x, torch.float16, 'x')
    b, h, w, c = x.shape
    out = torch.empty_like(x) if out is None else out
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_avgpool3x3_s1_excl_f16(_p(x), _p(out), b, h, w, c, _s()), 'yb_avgpool3x3_s1_excl_f16')
    return out


def avgpool3x3_s1_excl_bwd(dy, out=None):
    """Backward of avgpool3x3_s1_excl on fp16 NHWC dy [B,H,W,C]: each output's gradient divided by its own in-range count, gathered at the
    inputs of its window (fp32 sum, one rounding)."""
    _req(dy, torch.float16, 'dy')
    b, h, w, c = dy.shape
    out = torch.empty_like(dy) if out is None else out
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_avgpool3x3_s1_excl_bwd_f16(_p(dy), _p(out), b, h, w, c, _s()), 'yb_avgpool3x3_s1_excl_bwd_f16')
    return out


def conv2d_wgrad(x, dz, kh, kw, stride=1, pad=(0, 0), cin=None, cout=None, out=None):
    """yb_conv2d_wgrad: fp32 [Cout,kh,kw,Cin] (not scaled) of the yb_conv2d_bn_act_fwd geometry, from x fp16 [B,H,W,x_ld] (channels [0, cin))
    and dz fp16 [B,OH,OW,dz_ld] (channels [0, cout)) at the conv's output grid."""
    _req(x, torch.float16, 'x'); _req(dz, torch.float16, 'dz')
    b, h, wd, x_ld = x.shape
    cin = x_ld if cin is None else cin
    cout = dz.shape[-1] if cout is None else cout
    if tuple(dz.shape[:3]) != (b, conv2d_out_size(h, kh, stride, pad[0]), conv2d_out_size(wd, kw, stride, pad[1])):
        raise ValueError('conv2d_wgrad: dz %s is not the output grid of x %s' % (tuple(dz.shape), tuple(x.shape)))
    out = torch.empty(cout, kh, kw, cin, dtype=torch.float32, device=x.device) if out is None else _req(out, torch.float32, 'out')
    _ck(_l.load().yb_conv2d_wgrad(_p(x), _p(dz), _p(out), b, h, wd, cin, cout, kh, kw, stride, pad[0], pad[1], x_ld, dz.shape[-1], _s()),
        'yb_conv2d_wgrad')
    return out


def pack_weight_dgrad_khw_f16(w, cout_pad=None, cin_pad=None, out=None):
    """[Cout,Cin,kh,kw] fp32 -> fp16 [cin_pad,kh,kw,cout_pad]: rotated by 180 degrees, transposed, zero in the padding (the data-gradient operand)."""
    _req(w, torch.float32, 'weight')
    cout, cin, kh, kw = w.shape
    cout_pad = cout if cout_pad is None else cout_pad
    cin_pad = cin if cin_pad is None else cin_pad
    out = torch.empty(cin_pad, kh, kw, cout_pad, dtype=torch.float16, device=w.device) if out is None else out
    _ck(_l.load().yb_pack_weight_dgrad_khw_f16(_p(w), _p(out), cout, cin, kh, kw, cout_pad, cin_pad, _s()), 'yb_pack_weight_dgrad_khw_f16')
    return out


def stem3x3_s2_raw(x, w, pad=0):
    """Raw nn.Conv2d(3, 32, 3, stride 2, pad) (no BatchNorm, no ReLU): x fp32 NCHW [B,3,H,W] -> z fp16 NHWC [B,OH,OW,32]."""
    _req(x, torch.float32, 'x'); _req(w, torch.float32, 'w')
    b, c, h, wd = x.shape
    if c != 3 or tuple(w.shape) != (32, 3, 3, 3):
        raise ValueError('stem3x3_s2_raw: x [B,3,H,W] and w [32,3,3,3] expected')
    out = torch.empty(b, conv2d_out_size(h, 3, 2, pad), conv2d_out_size(wd, 3, 2, pad), 32, dtype=torch.float16, device=x.device)
    _ck(_l.load().yb_stem3x3_s2_raw_fwd(_p(x), _p(w), _p(out), b, h, wd, pad, _s()), 'yb_stem3x3_s2_raw_fwd')
    return out


def stem3x3_s2_wgrad(x, dz, pad=0, out=None):
    """Weight gradient of the stride-2 3 -> 32 stem: fp32 OIHW [32,3,3,3] from the fp32 NCHW image and dz fp16 NHWC [B,OH,OW,32]."""
    _req(x, torch.float32, 'x'); _req(dz, torch.float16, 'dz')
    b, _, h, wd = x.shape
    if tuple(dz.shape) != (b, conv2d_out_size(h, 3, 2, pad), conv2d_out_size(wd, 3, 2, pad), 32):
        raise ValueError('stem3x3_s2_wgrad: dz %s does not match x %s' % (tuple(dz.shape), tuple(x.shape)))
    out = torch.empty(32, 3, 3, 3, dtype=torch.float32, device=x.device) if out is None else out
    _ck(_l.load().yb_stem3x3_s2_wgrad(_p(x), _p(dz), _p(out), b, h, wd, pad, _s()), 'yb_stem3x3_s2_wgrad')
    return out


def maxpool3x3_s2_valid_bwd(x, dy, dy_ch_off=0, out=None):
    """Backward of maxpool3x3_s2_valid: dx [B,H,W,C] from its input x and dy = channels [dy_ch_off, dy_ch_off + C) of [B,OH,OW,dy_ld]."""
    _req(x, torch.float16, 'x'); _req(dy, torch.float16, 'dy')
    b, h, w, c = x.shape
    out = torch.empty_like(x) if out is None else out
    _ck(_l.load().yb_maxpool3x3_s2_valid_bwd_f16(_p(x), _p(dy), dy.shape[-1], dy_ch_off, _p(out), b, h, w, c, _s()), 'yb_maxpool3x3_s2_valid_bwd_f16')
    return out


def join(terms, out=None):
    """The sum of 2..4 fp16 tensors of one shape, in fp32, rounded once (yb_join_f16)."""
    if not 2 <= len(terms) <= 4:
        raise ValueError('join: 2 to 4 terms, got %d' % len(terms))
    for t in terms:
        _req(t, torch.float16, 'term')
        if t.shape != terms[0].shape:
            raise ValueError('join: shapes %s and %s differ' % (tuple(terms[0].shape), tuple(t.shape)))
    out = torch.empty_like(terms[0]) if out is None else out
    ts = list(terms) + [None] * (4 - len(terms))
    _ck(_l.load().yb_join_f16(*[_p(t) for t in ts], _p(out), out.numel(), _s()), 'yb_join_f16')
    return out


def conv1x1_preact(x, w, pre_scale, pre_shift, pre_relu, scale, shift, slope, out=None, out_mode=OUT_F16_NHWC, y_ch_off=0, cin=None, flags=0,
                   workspace=None):
    """DenseNet's norm -> relu -> 1x1 conv (yb_conv1x1_preact_fwd): the conv reads a = fp16(act(fmaf(pre_scale, x, pre_shift))) with act = ReLU
    (pre_relu) or identity, then applies the conv_bn_act epilogue (scale, shift, slope).  x: fp16 [B,H,W,x_ld] (the first `cin` channels,
    default the weight's Cin); w: fp16 [Cout,1,1,Cin]; out as conv_bn_act."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    _req(pre_scale, torch.float32, 'pre_scale'); _req(pre_shift, torch.float32, 'pre_shift')
    b, h, wd, x_ld = x.shape
    cout, k, _, wcin = w.shape
    cin = wcin if cin is None else cin
    if cin != wcin or k != 1:
        raise ValueError('conv1x1_preact: weight [%d,%d,%d,%d] does not match a 1x1 conv over %d channels' % (cout, k, k, wcin, cin))
    if pre_scale.numel() < cin or pre_shift.numel() < cin:
        raise ValueError('conv1x1_preact: pre_scale / pre_shift need %d channels' % cin)
    if out is None:
        out = (torch.empty(b, h, wd, cout, dtype=torch.float16, device=x.device) if out_mode == OUT_F16_NHWC
               else torch.empty(b, cout, h, wd, dtype=torch.float32, device=x.device))
    if out_mode == OUT_F16_NHWC:
        _req(out, torch.float16, 'out')
        y_ld = out.shape[-1]
    else:
        _req(out, torch.float32, 'out')
        y_ld = 0
    ws_ptr, ws_bytes = (None, 0) if workspace is None else (_p(_req(workspace, torch.uint8, 'workspace')), workspace.numel())
    _ck(_l.load().yb_conv1x1_preact_fwd(_p(x), _p(w), _p(pre_scale), _p(pre_shift), int(bool(pre_relu)), _p(scale), _p(shift), float(slope),
                                        _p(out), b, h, wd, cin, cout, x_ld, y_ld, y_ch_off, out_mode, flags, ws_ptr, ws_bytes, _s()),
        'yb_conv1x1_preact_fwd')
    return out


def conv1x1_preact_stats(x, w, pre_scale, pre_shift, pre_relu, sums, cin=None):
    """Training form of conv1x1_preact (yb_conv1x1_preact_stats_fwd): the raw output z = a . W^T (fp16 NHWC [B,H,W,Cout]) and, added into
    `sums` (float64 [2*Cout]), the per-channel sum and sum of squares of the stored values."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(pre_scale, torch.float32, 'pre_scale'); _req(pre_shift, torch.float32, 'pre_shift')
    _req(sums, torch.float64, 'sums')
    b, h, wd, x_ld = x.shape
    cout, k, _, wcin = w.shape
    cin = wcin if cin is None else cin
    if cin != wcin or k != 1 or sums.numel() != 2 * cout or pre_scale.numel() < cin or pre_shift.numel() < cin:
        raise ValueError('conv1x1_preact_stats: weight [%d,%d,%d,%d], %d input channels, %d sums' % (cout, k, k, wcin, cin, sums.numel()))
    one = torch.ones(cout, dtype=torch.float32, device=x.device)
    out = torch.empty(b, h, wd, cout, dtype=torch.float16, device=x.device)
    _ck(_l.load().yb_conv1x1_preact_stats_fwd(_p(x), _p(w), _p(pre_scale), _p(pre_shift), int(bool(pre_relu)), _p(one), _p(one.new_zeros(cout)), 1.0,
                                              _p(out), b, h, wd, cin, cout, x_ld, cout, 0, _p(sums), _s()), 'yb_conv1x1_preact_stats_fwd')
    return out


def conv1x1_preact_wgrad(x, pre_scale, pre_shift, pre_relu, dz, cin, cout):
    """Weight gradient of the pre-activation 1x1 conv (yb_conv1x1_preact_wgrad): fp32 [Cout,1,1,Cin] (yb_conv_wgrad's layout) from x fp16
    [B,H,W,x_ld] (channels [0, cin)) and dz fp16 [B,H,W,dz_ld]."""
    _req(x, torch.float16, 'x'); _req(dz, torch.float16, 'dz'); _req(pre_scale, torch.float32, 'pre_scale'); _req(pre_shift, torch.float32, 'pre_shift')
    b, h, wd, x_ld = x.shape
    dw = torch.empty(cout, 1, 1, cin, dtype=torch.float32, device=x.device)
    _ck(_l.load().yb_conv1x1_preact_wgrad(_p(x), _p(pre_scale), _p(pre_shift), int(bool(pre_relu)), _p(dz), _p(dw), b, h, wd, cin, cout, x_ld,
                                          dz.shape[-1], _s()), 'yb_conv1x1_preact_wgrad')
    return dw


def bn_batch_fold(mean, invstd, gamma, beta):
    """(scale, shift) of a train-mode pre-activation norm from the shared batch statistics (yb_bn_batch_fold)."""
    c = gamma.numel()
    scale = torch.empty(c, dtype=torch.float32, device=gamma.device)
    shift = torch.empty_like(scale)
    call('yb_bn_batch_fold', mean, invstd, gamma, beta, scale, shift, c)
    return scale, shift


def bn_preact_bwd(mode, x, mean, invstd, gamma, beta, relu, da, pool, sums, dx=None, dx16=None, dx16_ch0=0, channels=None):
    """One pass of a pre-activation norm's backward (yb_bn_preact_bwd) over channels [0, C) of x fp16 [B,H,W,x_ld]: mode 0 adds into `sums`
    (float64 [2C]); mode 1 adds dx into `dx` (fp32 [B,H,W,dx_ld]) and stores channels [dx16_ch0, C) of the result into `dx16` (fp16)."""
    b, h, wd, x_ld = x.shape
    c = gamma.numel() if channels is None else channels
    call('yb_bn_preact_bwd', int(mode), x, x_ld, mean, invstd, gamma, beta, int(relu), da, da.shape[-1], int(pool), b, h, wd, c, sums,
         dx, 0 if dx is None else dx.shape[-1], dx16, 0 if dx16 is None else dx16.shape[-1], int(dx16_ch0))


def conv_bn_act_split(x, w, scale, shift, slope, out, a_channels, y_ch_off=0, lo_ch_off=-1, out_mode=OUT_F16_NHWC, flags=0, workspace=None):
    """Split-precision conv unit (yb_conv_bn_act_split_fwd).  x: fp16 [B,H,W,x_ld] holding `a_channels` usable channels
    (C, or 2C = [hi | lo]); w: fp16 [Cout,k,k,K'] from pack_weight_split_f16; out fp16 [B,H,W,y_ld]: hi at y_ch_off, and the fp16
    rounding residual at lo_ch_off when lo_ch_off >= 0; or out fp32 [B,Cout,H,W]."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    b, h, wd, x_ld = x.shape
    cout, k, _, kch = w.shape
    if out_mode == OUT_F16_NHWC:
        _req(out, torch.float16, 'out')
        y_ld = out.shape[-1]
    else:
        _req(out, torch.float32, 'out')
        y_ld = 0
    ws_ptr, ws_bytes = (None, 0) if workspace is None else (_p(_req(workspace, torch.uint8, 'workspace')), workspace.numel())
    _ck(_l.load().yb_conv_bn_act_split_fwd(_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, kch, int(a_channels), cout, k, x_ld,
                                           y_ld, y_ch_off, lo_ch_off, out_mode, flags, ws_ptr, ws_bytes, _s()), 'yb_conv_bn_act_split_fwd')
    return out


def maxpool2x2_split(x, channels, out):
    """nn.MaxPool2d(2) on [hi | lo] activations: x [B,H,W,2C] -> out [B,H/2,W/2,2C]."""
    _req(x, torch.float16, 'x'); _req(out, torch.float16, 'out')
    b, h, w, x_ld = x.shape
    _ck(_l.load().yb_maxpool2x2_split_f16(_p(x), _p(out), b, h, w, channels, x_ld, channels, out.shape[-1], channels, _s()), 'yb_maxpool2x2_split_f16')
    return out


def conv_bn_act_stats(x, w, scale, shift, slope, sums, out=None, flags=0):
    """conv_bn_act (fp16 NHWC out) that also accumulates per-channel sum / sum of squares of the stored outputs into
    `sums` (float64 [2*Cout], zero on entry) in its epilogue -- the training forward's batch statistics."""
    _req(x, torch.float16, 'x'); _req(w, torch.float16, 'w'); _req(scale, torch.float32, 'scale'); _req(shift, torch.float32, 'shift')
    _req(sums, torch.float64, 'sums')
    b, h, wd, x_ld = x.shape
    cout, k, _, cin = w.shape
    if sums.numel() != 2 * cout:
        raise ValueError('sums must hold 2 * Cout doubles')
    if out is None:
        out = torch.empty(b, h, wd, cout, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_conv_bn_act_stats_fwd(_p(x), _p(w), _p(scale), _p(shift), float(slope), _p(out), b, h, wd, cin, cout, k, x_ld, out.shape[-1], 0,
                                           flags, _p(sums), _s()), 'yb_conv_bn_act_stats_fwd')
    return out


def maxpool2x2(x, channels=None, out=None):
    _req(x, torch.float16, 'x')
    b, h, w, x_ld = x.shape
    c = x_ld if channels is None else channels
    if out is None:
        out = torch.empty(b, h // 2, w // 2, c, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_maxpool2x2_f16(_p(x), _p(out), b, h, w, c, x_ld, _s()), 'yb_maxpool2x2_f16')
    return out


def maxpool2x2_s1(x, out=None):
    """ConstantPad2d((0,1,0,1), -inf) + MaxPool2d(2, stride=1) of model.yolo2.Tiny: fp16 NHWC, same spatial size."""
    _req(x, torch.float16, 'x')
    b, h, w, c = x.shape
    if out is None:
        out = torch.empty_like(x)
    _req(out, torch.float16, 'out')
    _ck(_l.load().yb_maxpool2x2_s1_f16(_p(x), _p(out), b, h, w, c, c, _s()), 'yb_maxpool2x2_s1_f16')
    return out


def reorg_f16(x, out, y_ch_off=0, channels=None, x_ch_off=0):
    """space-to-depth(2) of channels [x_ch_off, x_ch_off + channels) of x into channels [y_ch_off, y_ch_off + 4*channels) of out."""
    _req(x, torch.float16, 'x'); _req(out, torch.float16, 'out')
    b, h, w, x_ld = x.shape
    c = x_ld if channels is None else channels
    if x_ch_off % 8 or x_ch_off + c > x_ld:
        raise ValueError('reorg: bad channel slice')
    xp = ctypes.c_void_p(x.data_ptr() + 2 * x_ch_off)
    _ck(_l.load().yb_reorg_f16(xp, _p(out), b, h, w, c, x_ld, out.shape[-1], y_ch_off, _s()), 'yb_reorg_f16')
    return out


def reorg_f32_nchw(x, stride_h=2, stride_w=2):
    _req(x, torch.float32, 'x')
    b, c, h, w = x.shape
    out = torch.empty(b, c * stride_h * stride_w, h // stride_h, w // stride_w, dtype=torch.float32, device=x.device)
    if out.numel():
        _ck(_l.load().yb_reorg_f32_nchw(_p(x), _p(out), b, c, h, w, stride_h, stride_w, _s()), 'yb_reorg_f32_nchw')
    return out


def decode(feature, anchors, num_cls, with_prob=True):
    """feature fp32 [B,A*(5+C),rows,cols] -> dict(iou, center_offset, size_norm, yx_min, yx_max[, logits, prob])."""
    _req(feature, torch.float32, 'feature'); _req(anchors, torch.float32, 'anchors')
    b, ch, rows, cols = feature.shape
    a = anchors.shape[0]
    cells = rows * cols
    dev = feature.device
    out = dict(
        iou=torch.empty(b, cells, a, dtype=torch.float32, device=dev),
        center_offset=torch.empty(b, cells, a, 2, dtype=torch.float32, device=dev),
        size_norm=torch.empty(b, cells, a, 2, dtype=torch.float32, device=dev),
        yx_min=torch.empty(b, cells, a, 2, dtype=torch.float32, device=dev),
        yx_max=torch.empty(b, cells, a, 2, dtype=torch.float32, device=dev),
    )
    logits = prob = None
    if num_cls > 1:
        logits = out['logits'] = torch.empty(b, cells, a, num_cls, dtype=torch.float32, device=dev)
    if with_prob:
        prob = out['prob'] = torch.empty(b, cells, a, max(num_cls, 1), dtype=torch.float32, device=dev)
    if ch != a * (5 + (num_cls if num_cls > 1 else 0)):
        raise ValueError('feature has %d channels, expected %d' % (ch, a * (5 + (num_cls if num_cls > 1 else 0))))
    _ck(_l.load().yb_decode_fwd(_p(feature), _p(anchors), _p(out['iou']), _p(out['center_offset']), _p(out['size_norm']),
                                     _p(out['yx_min']), _p(out['yx_max']), _p(logits), _p(prob), b, rows, cols, a, num_cls, _s()),
             'yb_decode_fwd')
    return out


def filter_nms(score, yx_min, yx_max, prob, mode, threshold, threshold_cls, overlap, limit=200, expand=False, details=False):
    """Batched filter + NMS (+ per-class expansion).  score [B,n], yx_* [B,n,2], prob [B,n,C] or None.
    Returns a dict of int32/float32 device tensors (see include/yolo2_b200.h: yb_filter_nms)."""
    _req(score, torch.float32, 'score'); _req(yx_min, torch.float32, 'yx_min'); _req(yx_max, torch.float32, 'yx_max')
    if prob is not None:
        _req(prob, torch.float32, 'prob')
    b, n = score.shape
    num_cls = prob.shape[-1] if prob is not None else 1
    dev = score.device
    i32 = dict(dtype=torch.int32, device=dev)
    # every count is written by the image's CTA on every path (csrc/nms.cu), so no zero-fill launches precede the kernel
    res = dict(n_filtered=torch.empty(b, **i32), n_keep=torch.empty(b, **i32),
               keep_idx=torch.empty(b, limit, **i32), keep_box=torch.empty(b, limit, **i32))
    n_det = det_keep = det_cls = det_score = None
    det_cap = 0
    if expand:
        det_cap = limit * num_cls
        n_det = res['n_det'] = torch.empty(b, **i32)
        det_keep = res['det_keep'] = torch.empty(b, det_cap, **i32)
        det_cls = res['det_cls'] = torch.empty(b, det_cap, **i32)
        det_score = res['det_score'] = torch.empty(b, det_cap, dtype=torch.float32, device=dev)
    filt_box = best_cls = best_prob = None
    if details:
        filt_box = res['filt_box'] = torch.empty(b, n, **i32)
        if prob is not None:
            best_cls = res['best_cls'] = torch.empty(b, n, **i32)
            best_prob = res['best_prob'] = torch.empty(b, n, dtype=torch.float32, device=dev)
    _ck(_l.load().yb_filter_nms(_p(score), _p(yx_min), _p(yx_max), _p(prob), b, n, num_cls, mode, float(threshold),
                                     float(threshold_cls), float(overlap), limit, _p(res['n_filtered']), _p(res['n_keep']),
                                     _p(res['keep_idx']), _p(res['keep_box']), _p(n_det), _p(det_keep), _p(det_cls), _p(det_score),
                                     det_cap, _p(filt_box), _p(best_cls), _p(best_prob), _s()), 'yb_filter_nms')
    return res


def iou_matrix(yx_min1, yx_max1, yx_min2, yx_max2, min_union=1.1920928955078125e-07):
    """[N1,2]x2,[N2,2]x2 -> [N1,N2]  or batched [B,N1,2]... -> [B,N1,N2]."""
    for n, t in (('yx_min1', yx_min1), ('yx_max1', yx_max1), ('yx_min2', yx_min2), ('yx_max2', yx_max2)):
        _req(t, torch.float32, n)
    batched = yx_min1.dim() == 3
    b = yx_min1.shape[0] if batched else 1
    n1, n2 = yx_min1.shape[-2], yx_min2.shape[-2]
    out = torch.empty((b, n1, n2) if batched else (n1, n2), dtype=torch.float32, device=yx_min1.device)
    _ck(_l.load().yb_iou_matrix(_p(yx_min1), _p(yx_max1), _p(yx_min2), _p(yx_max2), _p(out), b, n1, n2, float(min_union), _s()),
             'yb_iou_matrix')
    return out


def region_loss_forward(feature, anchors, gt_yx_min, gt_yx_max, gt_cls, threshold, cross_entropy=True):
    """Region loss values + unweighted per-term gradients (see include/yolo2_b200.h: yb_region_loss_fwd).
    Returns dict(losses[5], positive, negative, best_iou, grad_terms, grad_bg)."""
    _req(feature, torch.float32, 'feature'); _req(anchors, torch.float32, 'anchors')
    _req(gt_yx_min, torch.float32, 'gt_yx_min'); _req(gt_yx_max, torch.float32, 'gt_yx_max')
    b, ch, rows, cols = feature.shape
    a = anchors.shape[0]
    per = ch // a
    num_cls = per - 5 if per > 5 else 1
    g = gt_yx_min.shape[1]
    if num_cls > 1:
        _req(gt_cls, torch.int64, 'gt_cls')
    cells = rows * cols
    dev = feature.device
    out = dict(losses=torch.empty(5, dtype=torch.float32, device=dev),
               positive=torch.empty(b, cells, a, dtype=torch.uint8, device=dev),
               negative=torch.empty(b, cells, a, dtype=torch.uint8, device=dev),
               best_iou=torch.empty(b, cells, a, dtype=torch.float32, device=dev),
               grad_terms=torch.empty_like(feature),
               grad_bg=torch.empty(b, a, cells, dtype=torch.float32, device=dev))
    pos_count = torch.empty(b, dtype=torch.int32, device=dev)
    partial = torch.empty(b * 5, dtype=torch.float32, device=dev)
    _ck(_l.load().yb_region_loss_fwd(_p(feature), _p(anchors), _p(gt_yx_min), _p(gt_yx_max), _p(gt_cls if num_cls > 1 else None), b, rows,
                                     cols, a, num_cls, g, float(threshold), int(bool(cross_entropy)), _p(out['losses']),
                                     _p(out['positive']), _p(out['negative']), _p(out['best_iou']), _p(pos_count), _p(partial),
                                     _p(out['grad_terms']), _p(out['grad_bg']), _s()), 'yb_region_loss_fwd')
    out['pos_count'] = pos_count
    return out


def region_loss_backward(grad_terms, grad_bg, weights5, num_anchors):
    """dfeature = sum_k weights5[k] * dloss_k/dfeature (weights5: device float32[5])."""
    _req(grad_terms, torch.float32, 'grad_terms'); _req(grad_bg, torch.float32, 'grad_bg'); _req(weights5, torch.float32, 'weights5')
    b, ch, rows, cols = grad_terms.shape
    per = ch // num_anchors
    num_cls = per - 5 if per > 5 else 1
    out = torch.empty_like(grad_terms)
    _ck(_l.load().yb_region_loss_bwd(_p(grad_terms), _p(grad_bg), _p(weights5), _p(out), b, rows, cols, num_anchors, num_cls, _s()),
        'yb_region_loss_bwd')
    return out


def call(name, *args):
    """Generic C-ABI call: tensors become device pointers (None -> NULL), the current stream is appended."""
    conv = [(_p(a) if isinstance(a, torch.Tensor) or a is None else a) for a in args]
    _ck(getattr(_l.load(), name)(*conv, _s()), name)
