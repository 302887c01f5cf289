"""The ping-pong consumer schedule of the wgmma convolution engine (each consumer warpgroup owns whole 128-row tiles,
the two alternate) against the cooperative one (both consumers split every tile).  Each output row gets the same
wgmma sequence and the same epilogue arithmetic, so the results must be bit-identical.  `engine` of conv_test: the
units digit picks the path (0 = what the network would take, 2 = per-tap, 3 = halo), the tens digit the schedule
(1 = cooperative, 2 = ping-pong)."""
import pytest
import torch

from test_gpu_conv import _case
from test_gpu_conv_halo import HALO_SHAPES

pytestmark = pytest.mark.gpu

COOP, PINGPONG = 10, 20


def _pair(x, w, bn, res, stride, relu, mode, path):
    from shapy_b200 import ops
    kw = dict(bn=bn, stride=stride, res_nhwc=res, relu=relu, mode=mode)
    return (ops.conv_test(x, w, engine=COOP + path, **kw), ops.conv_test(x, w, engine=PINGPONG + path, **kw))


@pytest.mark.parametrize('mode', [1, 0])
@pytest.mark.parametrize('shape', HALO_SHAPES)
def test_pingpong_halo(shape, mode):
    cin, cout, H, W, B = shape
    x, w, bn, res = _case(cin, cout, 3, 1, H, W, B, seed=6)
    y_coop, y_pp = _pair(x, w, bn, res, 1, True, mode, 3)
    assert torch.equal(y_pp, y_coop)


# (cin, cout, k, stride, H, W, B): 1x1 layers, stride-2 layers, a 3x3 stride-1 layer on the per-tap path, and the 7x7
# maps the network runs per-tap (several images per tile)
PER_TAP_SHAPES = [
    (64, 256, 1, 1, 56, 56, 2), (256, 64, 1, 1, 56, 56, 2), (96, 48, 1, 1, 28, 28, 3),
    (48, 96, 3, 2, 56, 56, 2), (96, 192, 3, 2, 28, 28, 3), (192, 384, 3, 2, 14, 14, 4),
    (48, 48, 3, 1, 56, 56, 2), (384, 384, 3, 1, 7, 7, 6),
]


@pytest.mark.parametrize('mode', [1, 0])
@pytest.mark.parametrize('shape', PER_TAP_SHAPES)
def test_pingpong_per_tap(shape, mode):
    cin, cout, k, stride, H, W, B = shape
    x, w, bn, res = _case(*shape, seed=7)
    y_coop, y_pp = _pair(x, w, bn, res, stride, True, mode, 2)
    assert torch.equal(y_pp, y_coop)


@pytest.mark.parametrize('relu', [False, True])
@pytest.mark.parametrize('with_res', [False, True])
@pytest.mark.parametrize('path', [2, 3])
def test_pingpong_epilogue_variants(path, with_res, relu):
    x, w, bn, res = _case(48, 48, 3, 1, 28, 28, 3, seed=8)
    y_coop, y_pp = _pair(x, w, bn, res if with_res else None, 1, relu, 1, path)
    assert torch.equal(y_pp, y_coop)


# tiles per CTA: one (a single image of 8 rows in two bands: two CTAs with one tile each, the second consumer idle),
# an odd count (280 halo tiles on 94 CTAs: three or two each), and many
@pytest.mark.parametrize('shape', [(48, 48, 8, 24, 1), (48, 48, 56, 56, 10), (96, 96, 28, 28, 33)])
def test_pingpong_tile_counts(shape):
    cin, cout, H, W, B = shape
    x, w, bn, res = _case(cin, cout, 3, 1, H, W, B, seed=9)
    for path in (2, 3):
        y_coop, y_pp = _pair(x, w, bn, res, 1, True, 1, path)
        assert torch.equal(y_pp, y_coop), path
