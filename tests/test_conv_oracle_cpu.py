"""The convolution oracle's error bound (tests/conv_oracle.py) against a small fp32 simulation of the wgmma kernel's
arithmetic: exact products, each k16 partial rounded once into an fp32 accumulator in tap-major order, the epilogue
in fp32, the output split-stored.  The simulation must pass the bound, and each seeded fault must fail it:

  drop_xl_wh_block   the xl.wh term of one 16-channel column block dropped (split mode)
  res_lo_missing     the residual's lo plane not added (split mode)
  skip_k16           one k16 step skipped
  bias_swap          the biases of two adjacent channels swapped
  relu_before_res    the ReLU applied before the residual add
  row_shift          one output row shifted by one pixel

The case gives output channels 16..31 weights 64x smaller than the rest, as BN folding does to a channel block with
a small gamma.  The checks these tests replace compared max|y - ref| / max|ref| < 2e-5 against an fp32 convolution
of the unsplit operands (split mode), and |y - ref| / (|ref| + 1e-2) < 1.2e-3 against one of the fp16-rounded
operands (fp16 mode).  OLD_CATCHES records which faults they catch on this case: they miss the dropped xl.wh block,
an error of ~2^-12 of that block's elements, which are small next to the tensor's maximum; the per-element bound
rejects it by 1.6-24x (and every other fault by 20x or more)."""
import pytest
import torch
import torch.nn.functional as F

import conv_oracle as co

# (cin, cout, k, stride, H, W, B)
SHAPES = [(32, 48, 3, 1, 6, 7, 2), (48, 32, 3, 2, 8, 6, 1), (64, 32, 1, 1, 5, 5, 2)]
FAULTS = ['drop_xl_wh_block', 'res_lo_missing', 'skip_k16', 'bias_swap', 'relu_before_res', 'row_shift']
SPLIT_ONLY = {'drop_xl_wh_block', 'res_lo_missing'}
SMALL = slice(16, 32)        # the output channel block with small weights, where the xl.wh fault is seeded

# (mode, fault) -> whether the old max-normalised / fp16-ulp check catches it on SHAPES[0]
OLD_CATCHES = {
    (1, 'drop_xl_wh_block'): False, (1, 'res_lo_missing'): True, (1, 'skip_k16'): True, (1, 'bias_swap'): True,
    (1, 'relu_before_res'): True, (1, 'row_shift'): True,
    (0, 'skip_k16'): True, (0, 'bias_swap'): True, (0, 'relu_before_res'): True, (0, 'row_shift'): True,
}


def _case(cin, cout, k, stride, H, W, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, cin, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    w[SMALL] /= 64
    bn = dict(weight=torch.rand(cout, generator=g) + 0.5, bias=torch.randn(cout, generator=g) * 0.1,
              mean=torch.randn(cout, generator=g) * 0.1, var=torch.rand(cout, generator=g) + 0.5, eps=1e-5)
    Ho, Wo = (H // 2, W // 2) if stride == 2 else (H, W)
    res = torch.randn(B, Ho, Wo, cout, generator=g)
    return x, w, bn, res


def simulate(x, weight, bn, stride, res, relu, mode, fault=None):
    """The kernel's arithmetic in fp32: (B, Ho, Wo, cout) as the library returns it (hi + lo / 2048)."""
    cout, cin, k, _ = weight.shape
    taps = k * k
    wf, b = co.fold(weight, None, bn)
    wh, wl = co.split(wf, mode)
    xh, xl = co.split(x, mode)
    B, H, W, _ = x.shape
    Ho, Wo = (H // 2, W // 2) if stride == 2 else (H, W)

    def cols(t):      # (B, cin, taps, L)
        return F.unfold(t.permute(0, 3, 1, 2), k, padding=k // 2, stride=stride).reshape(B, cin, taps, -1)
    ah = cols(xh)
    al = cols(xl) if mode else None
    bh, bl = wh.reshape(cout, cin, taps), (wl.reshape(cout, cin, taps) if mode else None)
    L = ah.shape[-1]
    d0, d1, d1p = (torch.zeros(B, L, cout, dtype=torch.float64) for _ in range(3))
    step, n = 0, taps * cin // 16
    for tap in range(taps):                     # tap-major, then k16 blocks: one fp32 rounding per partial
        for j in range(cin // 16):
            c = slice(16 * j, 16 * j + 16)
            if not (fault == 'skip_k16' and step == n // 2):
                d0 = co._f32(d0 + torch.einsum('bcl,oc->blo', ah[:, c, tap], bh[:, c, tap]))
                if mode:
                    d1 = co._f32(d1 + torch.einsum('bcl,oc->blo', ah[:, c, tap], bl[:, c, tap]))
                    d1p = co._f32(d1p + torch.einsum('bcl,oc->blo', al[:, c, tap], bh[:, c, tap]))
            step += 1
    if fault == 'drop_xl_wh_block':
        d1p[..., SMALL] = 0
    d0, d1, d1p = d0.float(), d1.float(), d1p.float()
    if fault == 'bias_swap':
        b = b.clone()
        b[[2, 3]] = b[[3, 2]]
    r = (d0 + (d1 + d1p) * co.LO if mode else d0) + b
    r = r.reshape(B, Ho, Wo, cout)
    if fault == 'relu_before_res':
        r = r.clamp_min(0)
    rh, rl = co.split(res, mode)
    r = r + rh.float()
    if mode and fault != 'res_lo_missing':
        r = r + rl.float() * co.LO
    if relu and fault != 'relu_before_res':
        r = r.clamp_min(0)
    hi, lo = co.split(r, mode)
    y = (hi + lo * co.LO if mode else hi).float()
    if fault == 'row_shift':
        y[0, 1, 1:] = y[0, 1, :-1].clone()
    return y


def _old_check(y, x, w, bn, stride, res, mode):
    """The checks the per-element bound replaces (see the module docstring): True if y passes."""
    x64, w64 = (x.double(), w.double()) if mode else (x.half().double(), None)
    s = bn['weight'].double() / torch.sqrt(bn['var'].double() + bn['eps'])
    shift = bn['bias'].double() - bn['mean'].double() * s
    if mode:
        ref = co._conv(x64, w64 * s[:, None, None, None], stride) + shift + res.double()
        ref = ref.clamp_min(0)
        return float((y.double() - ref).abs().max() / ref.abs().max()) < 2e-5
    wf, _ = co.fold(w, None, bn)
    ref = (co._conv(x64, wf.half().double(), stride) + shift + res.half().double()).clamp_min(0)
    return float(((y.double() - ref).abs() / (ref.abs() + 1e-2)).max()) < 1.2e-3


@pytest.mark.parametrize('mode', [1, 0])
@pytest.mark.parametrize('shape', SHAPES)
def test_simulated_kernel_within_bound(shape, mode):
    x, w, bn, res = _case(*shape)
    for with_res, relu in ((True, True), (False, True), (True, False)):
        r = res if with_res else None
        ref = co.reference(x, w, bn=bn, stride=shape[3], res=r, relu=relu, mode=mode)
        y = simulate(x, w, bn, shape[3], r if with_res else torch.zeros_like(res), relu, mode)
        assert co.ratio(y, ref) <= 1.0, (with_res, relu, co.ratio(y, ref))


@pytest.mark.parametrize('mode,fault', [(m, f) for m in (1, 0) for f in FAULTS if m or f not in SPLIT_ONLY])
@pytest.mark.parametrize('shape', SHAPES)
def test_seeded_fault_fails_bound(shape, mode, fault):
    x, w, bn, res = _case(*shape)
    ref = co.reference(x, w, bn=bn, stride=shape[3], res=res, relu=True, mode=mode)
    assert co.ratio(simulate(x, w, bn, shape[3], res, True, mode), ref) <= 1.0
    y = simulate(x, w, bn, shape[3], res, True, mode, fault)
    assert co.ratio(y, ref) > 1.0, co.ratio(y, ref)
    if shape == SHAPES[0]:
        assert (not _old_check(y, x, w, bn, shape[3], res, mode)) == OLD_CATCHES[(mode, fault)]
