"""The weight-resident halo path of the wgmma convolution engine (every CTA loads the layer's weights once, tiles load
only their halo band, operands in 16-channel slices) against the halo path of the same engine.  It issues the same
wgmmas in the same order with the same epilogue, so the results must be bit-identical.  `engine` of conv_test: units
digit 3 = halo, 4 = weight-resident; tens digit 1 = cooperative, 2 = ping-pong."""
import pytest
import torch

from test_gpu_conv import _case

pytestmark = pytest.mark.gpu

HALO, RESIDENT = 3, 4
SCHEDULES = [10, 20]   # cooperative, ping-pong


def _pair(x, w, bn, res, relu, mode, sched):
    from shapy_b200 import ops
    kw = dict(bn=bn, res_nhwc=res, relu=relu, mode=mode)
    return ops.conv_test(x, w, engine=sched + HALO, **kw), ops.conv_test(x, w, engine=sched + RESIDENT, **kw)


# c48 at 56^2: the bench batch (many tiles per CTA), B = 8, B = 3 (an odd tile count per CTA) and B = 1 (one tile per CTA)
@pytest.mark.parametrize('sched', SCHEDULES)
@pytest.mark.parametrize('mode', [1, 0])
@pytest.mark.parametrize('B', [64, 8, 3, 1])
def test_resident_c48(B, mode, sched):
    x, w, bn, res = _case(48, 48, 3, 1, 56, 56, B, seed=10)
    y_halo, y_res = _pair(x, w, bn, res, True, mode, sched)
    assert torch.equal(y_res, y_halo)


@pytest.mark.parametrize('relu', [False, True])
@pytest.mark.parametrize('with_res', [False, True])
@pytest.mark.parametrize('mode', [1, 0])
def test_resident_epilogue_variants(mode, with_res, relu):
    x, w, bn, res = _case(48, 48, 3, 1, 56, 56, 3, seed=11)
    for sched in SCHEDULES:
        y_halo, y_res = _pair(x, w, bn, res if with_res else None, relu, mode, sched)
        assert torch.equal(y_res, y_halo), sched


# other shapes the path holds: cin 16 / 32 / 64 slices, cout 64, a ragged last band and a non-square map
@pytest.mark.parametrize('shape', [(64, 64, 56, 56, 4, 0), (32, 48, 13, 24, 3, 1), (16, 64, 28, 28, 2, 1),
                                   (48, 48, 8, 24, 1, 1)])
def test_resident_shapes(shape):
    cin, cout, H, W, B, mode = shape
    x, w, bn, res = _case(cin, cout, 3, 1, H, W, B, seed=12)
    for sched in SCHEDULES:
        y_halo, y_res = _pair(x, w, bn, res, True, mode, sched)
        assert torch.equal(y_res, y_halo), sched


# what the network runs: the planner's choice for c48 (split and fp16) and for b64 in fp16 matches the halo path
@pytest.mark.parametrize('shape', [(48, 48, 1), (48, 48, 0), (64, 64, 0)])
def test_resident_planner_layers(shape):
    from shapy_b200 import ops
    cin, cout, mode = shape
    x, w, bn, res = _case(cin, cout, 3, 1, 56, 56, 8, seed=13)
    y_auto = ops.conv_test(x, w, bn=bn, res_nhwc=res, relu=True, mode=mode, engine=0)
    y_halo = ops.conv_test(x, w, bn=bn, res_nhwc=res, relu=True, mode=mode, engine=HALO)
    assert torch.equal(y_auto, y_halo)


# (cin, cout, k, stride, H, W, B, mode): cin past 64, cout 96, stride 2, 1x1, and split b64 (weights do not fit)
@pytest.mark.parametrize('shape', [(96, 96, 3, 1, 28, 28, 1, 1), (48, 96, 3, 1, 28, 28, 1, 0),
                                   (48, 96, 3, 2, 56, 56, 1, 1), (64, 64, 1, 1, 56, 56, 1, 0),
                                   (64, 64, 3, 1, 56, 56, 1, 1)])
def test_resident_rejects_other_layers(shape):
    """Forcing the resident path on a layer it cannot hold is an error, not a fall-back."""
    from shapy_b200 import ops
    cin, cout, k, stride, H, W, B, mode = shape
    x, w, bn, _ = _case(cin, cout, k, stride, H, W, B)
    with pytest.raises(RuntimeError):
        ops.conv_test(x, w, bn=bn, stride=stride, relu=True, mode=mode, engine=RESIDENT)
