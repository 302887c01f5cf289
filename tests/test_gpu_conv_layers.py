"""Every distinct wgmma convolution of HighResolutionNet.build_program(), at the bench configurations (224 x 224:
split fp16 at B = 64, plain fp16 at B = 32) and at the 256 x 256 and 64 x 96 inputs the end-to-end tests use, run
as the network plans it (engine 0) into the layer's real output view (its out_coff and channel count, which is 1536
for the slices of the concatenated tensor), against the float64 oracle's per-element bound (tests/conv_oracle.py).
Channels outside the slice and the guard image past the batch must stay NaN.  The plan the engine reports, forced
explicitly, must give the same bits: the planner's pick is one of the candidates test_gpu_conv_tiles.py checks."""
import functools

import pytest
import torch

import conv_oracle as co
from test_gpu_conv import _case

pytestmark = pytest.mark.gpu

# (H, W, B, mode)
CONFIGS = [(224, 224, 64, 1), (224, 224, 32, 0), (256, 256, 2, 1), (256, 256, 2, 0), (64, 96, 2, 1), (64, 96, 2, 0)]


@functools.lru_cache(maxsize=None)
def _program():
    from shapy_b200 import synth
    return synth.build_synthetic_regressor().backbone.build_program()[:3]


def layers(H, W):
    """Distinct (cin, cout, k, stride, H_in, W_in, in_ctot, out_ctot, out_coff, residual, relu) of the program's
    convolutions the wgmma engine runs (cin and cout multiples of 16; the rest run on the SIMT engine)."""
    from shapy_b200._lib import OP_CONV
    convs, ops, slots = _program()
    out = {}
    for o in ops:
        if o['kind'] != OP_CONV:
            continue
        c = convs[o['conv']]
        if c['cin'] % 16 or c['cout'] % 16:
            continue
        d = slots[o['in_slot']]['div']
        out[(c['cin'], c['cout'], c['ksize'], c['stride'], H // d, W // d, slots[o['in_slot']]['channels'],
             slots[o['out_slot']]['channels'], o['out_coff'], o['res_slot'] >= 0, bool(o['relu']))] = None
    return list(out)


@pytest.mark.parametrize('config', CONFIGS, ids=lambda c: f'{c[0]}x{c[1]}-b{c[2]}-mode{c[3]}')
def test_network_layers(config):
    from shapy_b200 import ops
    H0, W0, B, mode = config
    ls = layers(H0, W0)
    assert len(ls) > 30
    for i, (cin, cout, k, s, H, W, in_ctot, out_ctot, coff, with_res, relu) in enumerate(ls):
        x, w, bn, res = _case(cin, cout, k, s, H, W, B, seed=30 + i)
        res = res if with_res else None
        assert in_ctot == cin
        kw = dict(bn=bn, stride=s, res_nhwc=res, relu=relu, mode=mode, out_view=(out_ctot, coff))
        y, plan = ops.conv_test(x, w, engine=0, report=True, **kw)
        sl = y[:B, ..., coff:coff + cout]
        ref = co.reference(x, w, bn=bn, stride=s, res=res, relu=relu, mode=mode)
        r = co.ratio(sl, ref)
        what = f'{cin}->{cout} {k}x{k} s{s} @{H}x{W} B {B} mode {mode} view ({out_ctot}, {coff}) res {with_res}'
        print(f'[layers] {what}: {tuple(plan)} ratio {r:.3g}')
        assert r <= 1.0, (what, plan, co.worst(sl, ref))
        outside = torch.ones_like(y, dtype=torch.bool)
        outside[:B, ..., coff:coff + cout] = False
        assert y[outside].isnan().all(), what
        forced = ops.conv_test(x, w, engine=plan.engine, **kw)
        assert torch.equal(forced.view(torch.int32), y.view(torch.int32)), (what, plan)   # NaN guard included
