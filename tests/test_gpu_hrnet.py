"""HRNet-W48 through the C ABI against the reference module's own outputs on the seeded synthetic
checkpoint (tests/golden/ref_hrnet.npz) and against the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import net_oracle
from shapy_b200 import synth

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


@pytest.fixture(scope='module')
def backbone():
    return synth.build_synthetic_regressor().backbone


def _inputs():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 224, 224, generator=g)
    x64 = torch.randn(1, 3, 64, 96, generator=g)
    return x, x64


@pytest.mark.parametrize('engine', [1, 0])
def test_hrnet_vs_reference_golden(backbone, golden_dir, engine):
    g = np.load(os.path.join(golden_dir, 'ref_hrnet.npz'))
    x, x64 = _inputs()
    bb = backbone.cuda().eval()
    bb.engine, bb.precision_mode = engine, 1
    bb.invalidate()
    out = bb(x.cuda())
    assert rel(out['concat'], g['concat']) < 1e-4, rel(out['concat'], g['concat'])
    assert rel(out['layer1'][:, ::7, ::5, ::5], g['layer1_sub']) < 1e-4
    assert rel(out['layer4'][:, ::16], g['layer4']) < 1e-4
    out64 = bb(x64.cuda())                     # non-square, non-224 input: 16x24 ... 2x3 feature maps
    assert rel(out64['concat'], g['concat64']) < 1e-4


def test_hrnet_fp16_mode_close(backbone, golden_dir):
    """BASELINE config 2 numerics: single-pass fp16 operands (not the parity mode)."""
    g = np.load(os.path.join(golden_dir, 'ref_hrnet.npz'))
    x, _ = _inputs()
    bb = backbone.cuda().eval()
    bb.engine, bb.precision_mode = 0, 0
    bb.invalidate()
    out = bb(x.cuda())
    assert rel(out['concat'], g['concat']) < 3e-2
    bb.precision_mode = 1
    bb.invalidate()


def test_hrnet_batch_independence(backbone):
    """Images are independent: a permutation of the batch permutes the outputs bit for bit (same launch
    configuration), and a sub-batch matches to fp32 rounding (the tile configuration depends on the batch
    size, which changes the summation order)."""
    bb = backbone.cuda().eval()
    bb.engine, bb.precision_mode = 0, 1
    bb.invalidate()
    x = torch.randn(9, 3, 224, 224, generator=torch.Generator().manual_seed(5)).cuda()
    full = bb(x)['concat']
    perm = torch.tensor([4, 0, 8, 2, 6, 1, 7, 3, 5]).cuda()
    assert torch.equal(bb(x[perm].contiguous())['concat'], full[perm])
    part = bb(x[3:5].contiguous())['concat']
    assert rel(part, full[3:5]) < 1e-5


def rms_rel(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float(((a - b) ** 2).mean().sqrt() / (b ** 2).mean().sqrt())


def _backbone_sd(bb):
    return {k: v.detach().clone() for k, v in bb.state_dict().items()}


def test_hrnet_256x256_vs_oracle(backbone):
    """The reference's default crop (config/datasets_defaults.py:30): 64 / 32 / 16 / 8-wide maps, tile shapes the
    224 x 224 tests never run."""
    bb = backbone.cuda().eval()
    bb.engine, bb.precision_mode = 0, 1
    bb.invalidate()
    x = torch.randn(3, 3, 256, 256, generator=torch.Generator().manual_seed(11))
    sd = {k: v.cpu() for k, v in _backbone_sd(bb).items()}
    with torch.no_grad():
        ref = net_oracle.hrnet_forward(sd, x)
    out = bb(x.cuda())
    for k in ('layer1', 'layer2', 'layer3', 'layer4', 'concat'):
        assert rel(out[k], ref[k]) < 1e-4, (k, rel(out[k], ref[k]))
        assert rms_rel(out[k], ref[k]) < 5e-5, (k, rms_rel(out[k], ref[k]))


def test_hrnet_B64_224_rows_vs_oracle(backbone):
    """BASELINE configs[2] launch configuration (B = 64, 224 x 224): the tile shapes halo_configure picks depend on
    the batch, so the benchmarked configuration itself is checked; the oracle runs on 6 of the 64 images."""
    bb = backbone.cuda().eval()
    bb.engine, bb.precision_mode = 0, 1
    bb.invalidate()
    x = torch.randn(64, 3, 224, 224, generator=torch.Generator().manual_seed(12))
    rows = [0, 13, 31, 32, 50, 63]
    sd = {k: v.cpu() for k, v in _backbone_sd(bb).items()}
    with torch.no_grad():
        ref = net_oracle.hrnet_forward(sd, x[rows])
    out = bb(x.cuda())
    for k in ('layer1', 'layer2', 'layer3', 'layer4', 'concat'):
        mine = out[k][rows]
        assert rel(mine, ref[k]) < 1e-4, (k, rel(mine, ref[k]))
        assert rms_rel(mine, ref[k]) < 5e-5, (k, rms_rel(mine, ref[k]))


def test_hrnet_fp16_B32_vs_fp16_operand_reference(backbone):
    """BASELINE configs[1] (HRNet only, fp16, B = 32): every stage against a plain-PyTorch fp32 reference of the same
    arithmetic (BN folded, conv operands and stored activations rounded to fp16, fp32 accumulation; cuDNN, TF32 off).
    The two sides accumulate in different orders, so now and then an activation rounds to the neighbouring fp16 value;
    each such flip is as large as the rounding noise itself, so after ~110 layers the two fp16 realisations are as far
    from each other as either is from the fp32 network (measured: 1.1e-3 RMS, 2.5e-3 max on layer1).  The bars are
    therefore fp16-noise sized; the per-layer checks that cannot amplify are tests/test_gpu_conv_layers.py (every
    layer of this program, within a float64 per-element bound of half an fp16 ulp plus the accumulation error) and
    tests/test_gpu_conv.py::test_conv_fp16_benchmark_batch.  A wrong tile or a dropped tap here is O(1)."""
    bb = backbone.cuda().eval()
    bb.engine, bb.precision_mode = 0, 0
    bb.invalidate()
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        x = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(13)).cuda()
        sd = {k: v.cuda() for k, v in _backbone_sd(bb).items()}
        with torch.no_grad():
            ref = net_oracle.hrnet_forward(sd, x, rnd=lambda t: t.half().float())
        out = bb(x)
        for k in ('layer1', 'layer2', 'layer3', 'layer4', 'concat'):
            assert rel(out[k], ref[k]) < 2e-2, (k, rel(out[k], ref[k]))
            assert rms_rel(out[k], ref[k]) < 5e-3, (k, rms_rel(out[k], ref[k]))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
        bb.precision_mode = 1
        bb.invalidate()


_LANE_SCRIPT = r'''
import sys, torch
sys.path.insert(0, sys.argv[1])
from shapy_b200 import synth
bb = synth.build_synthetic_regressor().backbone.cuda().eval()
x = torch.randn(5, 3, 224, 224, generator=torch.Generator().manual_seed(31)).cuda()
outs = []
for _ in range(4):
    o = bb(x)
    outs.append(torch.cat([o['concat'].flatten(), o['layer1'].flatten(), o['layer4'].flatten()]).cpu())
assert all(torch.equal(outs[0], t) for t in outs[1:]), 'forward is not deterministic'
torch.save(outs[0], sys.argv[2])
'''


def test_lane_schedule_is_bit_identical_to_serial_execution(tmp_path):
    """The multi-lane executor (branches of a module on concurrent streams, cross-lane ordering derived from slot
    hazards) must give exactly the serial program's result: SHAPY_HRNET_LANES=1 vs the default 4 lanes, each run four
    times (a missing dependency would show up as run-to-run differences as well)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = {}
    for lanes in ('1', '4'):
        out = str(tmp_path / f'lanes{lanes}.pt')
        env = dict(os.environ, SHAPY_HRNET_LANES=lanes)
        r = subprocess.run([sys.executable, '-c', _LANE_SCRIPT, root, out], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        res[lanes] = torch.load(out)
    assert torch.equal(res['1'], res['4'])
