"""Float64 reference of one wgmma-engine convolution over the operands the device holds, with a per-element error
bound derived from the kernel's arithmetic (not fitted to observed errors).

Operands, bit for bit what the library stores:
  activations, residual   launch_nhwc_split / split_store: v = clamp(x, +-65504) in fp32, hi = fp16(v),
                          lo = fp16((v - hi) * 2048)  (v - hi is exact in fp32, * 2048 too)
  weights                 pack_conv: s = gamma / sqrt(var + eps), w * s in fp32 (BN folded), split as above
  bias                    pack_conv: (b - mean) * s + beta in fp32 (the conv bias alone without BN, else 0)
fp16 mode (mode 0) keeps the hi planes only.

Reference, in float64 (each product of two fp16 values is exact; a sum of a few thousand of them errs by ~2^-40 of
its absolute sum, far below every term of the bound):
  split:  R = relu(conv(xh, wh) + 2^-11 (conv(xh, wl) + conv(xl, wh)) + bias [+ rh + 2^-11 rl])
  fp16:   R = relu(conv(xh, wh) + bias [+ rh])
xl.wl is not a term: the kernel does not issue it.  A is the same expression over absolute values, without the ReLU.

Bound, |y - R| <= (s n + c) 2^-23 A + (output rounding), with n = taps * cin / 16, the k16 steps the kernel issues
for one output element.  Model of one k16 step of the tensor core (wgmma m64nNk16, fp16 operands, fp32 accumulator
D), measured on the H100 by test_gpu_conv_tiles.py::test_k16_step_model: the 16 products are exact; they and D are
aligned to the largest exponent e among them and each is truncated toward zero to a multiple of 2^(e - 25) (two bits
below the fp32 ulp of 2^e); the aligned terms are summed exactly and the sum is truncated to fp32.  The alignment
loses < 17 * 2^(e - 25) = 4.25 * 2^-23 * 2^e, the final truncation < 2^-23 |sum|, and both 2^e and |sum| are at
most |D| + sum |p| <= A, so a step errs by < s 2^-23 A with s = 5.25.  Over n steps: s n 2^-23 A (the running |D|
never exceeds A by more than a factor 1 + s n 2^-23).  A single truncation of the exact step sum (s = 1) is not
the hardware: with one dominant product per step and the other products just under the fp32 ulp, the device loses
a quarter ulp per product.  c = 4 covers the epilogue's fp32 additions, each rounded to nearest (<= 2^-24 A):
D0 + (D1 + D1') / 2048, + bias, + rh, + rl / 2048, and the 2^-11-scaled accumulation error of D1 and D1'.
Output rounding: split mode stores hi = fp16(v), lo = fp16((v - hi) 2048); lo keeps 11 bits of v - hi, itself
< 2^-11 |v|, so the pair errs by <= 2^-22 |v| (+ 2^-36 where lo is subnormal).  fp16 mode rounds v to fp16: half an
ulp, <= 2^-11 |v| (+ 2^-25 among subnormals).  |v| <= |R| + (the accumulation term), and the ReLU is 1-Lipschitz.
If a kernel ever exceeds this bound, revisit the model, not the constants.

The module runs on whichever device its inputs are on: float64 convolutions through torch.
"""
from typing import NamedTuple

import torch
import torch.nn.functional as F

STEP = 1 + 17 / 4    # error of one k16 step, in units of 2^-23 A (see above)
C_EPI = 4            # epilogue roundings, in units of 2^-23 A
LO = 2.0 ** -11      # weight of a lo plane


class Reference(NamedTuple):
    R: torch.Tensor      # float64 NHWC, the convolution over the stored operands
    A: torch.Tensor      # float64 NHWC, the same over absolute values (pre-ReLU)
    steps: int           # k16 steps per output element
    mode: int            # 1 split fp16, 0 plain fp16


def split(t, mode=1):
    """split_store of an fp32 tensor: (hi, lo) as float64 tensors of the stored fp16 values (lo None in fp16 mode)."""
    v = t.float().clamp(-65504.0, 65504.0)
    hi = v.half()
    lo = ((v - hi.float()) * 2048.0).half().double() if mode else None
    return hi.double(), lo


def _f32(t):
    return t.float().double()


def fold(weight, bias=None, bn=None):
    """pack_conv's BN folding in fp32, on the CPU: (w * s, bias), both fp32.  Each fp32 operation is done in float64
    and rounded once to fp32, which gives the correctly rounded fp32 result of a +, *, / or sqrt, as the host code
    computes it (torch's vectorised fp32 sqrt is not always correctly rounded)."""
    w = weight.detach().float().cpu()
    cout = w.shape[0]
    b = bias.detach().float().cpu() if bias is not None else torch.zeros(cout)
    if bn is None:
        return w, b
    g, beta, mean, var = (_f32(bn[k].detach().cpu()) for k in ('weight', 'bias', 'mean', 'var'))
    s = _f32(g / _f32(_f32(var + _f32(torch.tensor(bn['eps']))).sqrt()))
    shift = _f32(_f32(_f32(b.double() - mean) * s) + beta)
    return _f32(w.double() * s[:, None, None, None]).float(), shift.float()


def _conv(x, w, stride):
    return F.conv2d(x.permute(0, 3, 1, 2), w, stride=stride, padding=w.shape[-1] // 2).permute(0, 2, 3, 1)


def reference(x, weight, bias=None, bn=None, stride=1, res=None, relu=False, mode=1):
    """x (B, H, W, cin) fp32 NHWC and the arguments of ops.conv_test -> Reference."""
    dev = x.device
    wf, bf = fold(weight, bias, bn)
    wh, wl = (t.to(dev) if t is not None else None for t in split(wf, mode))
    xh, xl = split(x, mode)
    b = bf.double().to(dev)
    if mode:
        # one float64 convolution over [xh | xh | xl] x [wh | wl / 2048 | wh / 2048] (scaling by 2^-11 is exact)
        xs = torch.cat([xh, xh, xl], dim=3)
        ws = torch.cat([wh, wl * LO, wh * LO], dim=1)
    else:
        xs, ws = xh, wh
    del xh, xl
    pre = _conv(xs, ws, stride) + b
    A = _conv(xs.abs(), ws.abs(), stride) + b.abs()
    del xs
    if res is not None:
        rh, rl = split(res, mode)
        pre += rh
        A += rh.abs()
        if mode:
            pre += rl * LO
            A += rl.abs() * LO
    R = pre.clamp_min(0.0) if relu else pre
    k = weight.shape[-1]
    return Reference(R, A, k * k * (weight.shape[1] // 16), mode)


def bound(ref):
    acc = (STEP * ref.steps + C_EPI) * 2.0 ** -23 * ref.A
    v = ref.R.abs() + acc
    return acc + (2.0 ** -22 * v + 2.0 ** -36 if ref.mode else 2.0 ** -11 * v + 2.0 ** -25)


def ratio(y, ref):
    """max over elements of |y - R| / bound; inf where y is not finite."""
    r = (y.double() - ref.R).abs() / bound(ref)
    return float(torch.nan_to_num(r, nan=float('inf')).max()) if r.numel() else 0.0


def worst(y, ref):
    """The element of largest |y - R| / bound, for a failure message."""
    b = bound(ref)
    r = torch.nan_to_num((y.double() - ref.R).abs() / b, nan=float('inf'))
    i = int(r.flatten().argmax())
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape))
    return (f'worst at {idx}: y {float(y[idx]):.9g} R {float(ref.R[idx]):.9g} A {float(ref.A[idx]):.6g} '
            f'bound {float(b[idx]):.4g} ratio {float(r[idx]):.4g} ({ref.steps} k16 steps)')
