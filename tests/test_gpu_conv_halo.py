"""The halo-resident path of the wgmma convolution engine (3x3 stride-1 layers, one channel block loaded once with its
halo for all nine taps) against the per-tap path of the same engine and against cuDNN fp32.  `engine` of conv_test
picks the path: 2 = per-tap, 3 = halo, 0 = whatever the network would take."""
import pytest
import torch

from test_gpu_conv import _case, _ref, rel

pytestmark = pytest.mark.gpu

# (cin, cout, H, W, B): the BasicBlock families at the bench batch (224^2 input), the widths a 256^2 input gives, a
# map whose last band is ragged (13 rows in bands of 4), a non-square one, a cin that is not a multiple of 64, the
# transition layer, and a 7x7 map (which the network runs per-tap; the forced halo path must still be right)
HALO_SHAPES = [
    (48, 48, 56, 56, 64), (96, 96, 28, 28, 64), (192, 192, 14, 14, 64),
    (48, 48, 64, 64, 8), (96, 96, 32, 32, 8), (192, 192, 16, 16, 8),
    (48, 48, 13, 24, 3), (48, 48, 8, 24, 1), (160, 64, 20, 20, 2), (256, 48, 56, 56, 1), (384, 384, 7, 7, 5),
]


@pytest.mark.parametrize('shape', HALO_SHAPES)
def test_halo_matches_per_tap_split(shape):
    from shapy_b200 import ops
    cin, cout, H, W, B = shape
    x, w, bn, res = _case(cin, cout, 3, 1, H, W, B, seed=4)
    y_tap = ops.conv_test(x, w, bn=bn, res_nhwc=res, relu=True, mode=1, engine=2)
    y_halo = ops.conv_test(x, w, bn=bn, res_nhwc=res, relu=True, mode=1, engine=3)
    if cin <= 64:      # one channel block: the same wgmmas in the same order
        assert torch.equal(y_halo, y_tap)
    else:              # channel-block-major order: fp32 sums reordered
        assert rel(y_halo, y_tap) < 5e-6, rel(y_halo, y_tap)
    ref = _ref(x, w, None, bn, 1, res, True)
    assert rel(y_halo, ref) < 2e-5, rel(y_halo, ref)
    y_auto = ops.conv_test(x, w, bn=bn, res_nhwc=res, relu=True, mode=1, engine=0)
    assert rel(y_auto, ref) < 2e-5, rel(y_auto, ref)


@pytest.mark.parametrize('shape', HALO_SHAPES[:3] + HALO_SHAPES[6:7])
def test_halo_matches_per_tap_fp16(shape):
    from shapy_b200 import ops
    cin, cout, H, W, _ = shape
    x, w, bn, _ = _case(cin, cout, 3, 1, H, W, 32 if H >= 14 else 3, seed=5)
    y_tap = ops.conv_test(x, w, bn=bn, relu=True, mode=0, engine=2)
    y_halo = ops.conv_test(x, w, bn=bn, relu=True, mode=0, engine=3)
    if cin <= 64:
        assert torch.equal(y_halo, y_tap)
    else:              # outputs are fp16: a reordered fp32 sum may round to the neighbouring fp16 value
        err = (y_halo - y_tap).abs() / (y_tap.abs() + 1e-2)
        assert float(err.max()) < 1.2e-3, float(err.max())


@pytest.mark.parametrize('shape', [(48, 96, 3, 2, 56, 56, 1), (64, 256, 1, 1, 56, 56, 1)])
def test_halo_rejects_other_layers(shape):
    """Stride-2 and 1x1 layers have no halo path: forcing it is an error."""
    from shapy_b200 import ops
    cin, cout, k, stride, H, W, B = shape
    x, w, bn, _ = _case(*shape)
    with pytest.raises(RuntimeError):
        ops.conv_test(x, w, bn=bn, stride=stride, relu=True, mode=1, engine=3)
