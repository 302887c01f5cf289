"""shapy_mmi_forward_f64 (ops.mesh_to_mesh_forward on float64 triangles) on the GPU:
  - against the reference operator's own float64 results (tests/golden/ref_mmi_*_f64.npz), with the bars of
    tests/test_gpu_zz_reference_op.py: the reference build contracts multiply-adds into FMAs and this one does not, so
    a pair sitting exactly on a tolerance may fall on the other side;
  - against the double build of the C oracle (oracle/mmi_oracle_scalar.c, -DMMI_DOUBLE), bit for bit;
  - the call's contract: dtypes, shapes, empty sizes, refusals, determinism, batch independence, graph capture."""
import numpy as np
import pytest
import torch

from oracle import mmi_oracle_f64
from test_mmi_f64_cpu import (as_dict, check_quirk, compare, load_reference, plane_inputs_f64, quirk_inputs_f64,
                              soup_inputs_f64)

pytestmark = pytest.mark.gpu


def run(query, target, M):
    from shapy_b200 import ops
    f, b = ops.mesh_to_mesh_forward(torch.from_numpy(np.ascontiguousarray(query)).cuda(),
                                    torch.from_numpy(np.ascontiguousarray(target)).cuda(), M)
    assert f.dtype == torch.int64 and b.dtype == torch.float64
    return f.cpu().numpy(), b.cpu().numpy()


def test_plane_vs_reference(golden_dir):
    query, tris, M = plane_inputs_f64(golden_dir)
    ref_f, ref_b = load_reference('ref_mmi_plane_f64', query)
    f, b = run(query, tris, M)
    worst = 0.0
    for i in range(query.shape[0]):
        n, e = compare(as_dict(ref_f[i], ref_b[i], M), as_dict(f[i], b[i], M), 2, f'body {i}')
        assert n > 50
        worst = max(worst, e)
    print(f'plane f64: largest barycentric difference to the reference {worst:.2e}')


def test_soup_vs_reference():
    query, target, M = soup_inputs_f64()
    ref_f, ref_b = load_reference('ref_mmi_soup_f64', query)
    f, b = run(query, target, M)
    total, worst = 0, 0.0
    for i in range(query.shape[0]):
        r = as_dict(ref_f[i], ref_b[i], M)
        n, e = compare(r, as_dict(f[i], b[i], M), max(2, len(r) // 100), f'soup {i}')
        total, worst = total + n, max(worst, e)
    assert total > 100
    print(f'soup f64: largest barycentric difference to the reference {worst:.2e}')


def test_quirk_vs_reference():
    """Pairs that only the reference's float rounding in its double SAT reports: the sets must be identical."""
    query, target, M, pairs = quirk_inputs_f64()
    ref_f, ref_b = load_reference('ref_mmi_quirk_f64', query)
    f, b = run(query, target, M)
    check_quirk(f[0], M, pairs, 'shapy_mmi_forward_f64')
    compare(as_dict(ref_f[0], ref_b[0], M), as_dict(f[0], b[0], M), 0, 'quirk')


def _per_query(faces, bcs, Q, M):
    out = []
    for q in range(Q):
        fq, bq = faces[q * M:(q + 1) * M], bcs[q * M:(q + 1) * M]
        idx = np.nonzero(fq >= 0)[0]
        order = np.argsort(fq[idx], kind='stable')
        out.append((fq[idx][order], bq[idx][order]))
    return out


def assert_matches_oracle(query, target, M):
    """Each query's sorted face set and its barycentrics equal the double oracle's bit for bit.  A query with more than
    M collisions keeps an unspecified M of them: those must be oracle collisions with the oracle's barycentrics.
    Returns (collisions compared, overflowing queries)."""
    B, Q = query.shape[:2]
    f, b = run(query, target, M)
    M_all = min(target.shape[1], max(8 * M, 256))
    rf, rb = mmi_oracle_f64.mesh_to_mesh_forward(query, target, M_all)
    n_hits = n_over = 0
    for i in range(B):
        for q, ((f1, b1), (f2, b2)) in enumerate(zip(_per_query(f[i], b[i], Q, M), _per_query(rf[i], rb[i], Q, M_all))):
            assert len(f2) < M_all or M_all == target.shape[1], 'the oracle must see every collision'
            if len(f2) <= M:
                assert np.array_equal(f1, f2), (i, q)
                assert np.array_equal(b1, b2), (i, q)
            else:
                n_over += 1
                assert len(f1) == M and np.isin(f1, f2).all(), (i, q)
                assert np.array_equal(b1, b2[np.searchsorted(f2, f1)]), (i, q)
            n_hits += len(f1)
    return n_hits, n_over


def test_plane_vs_double_oracle_bit_exact(golden_dir):
    query, tris, M = plane_inputs_f64(golden_dir)
    assert assert_matches_oracle(query, tris, M)[0] > 200


def test_quirk_vs_double_oracle_bit_exact():
    query, target, M, _ = quirk_inputs_f64()
    assert assert_matches_oracle(query, target, M)[0] == 10


@pytest.mark.parametrize('Q,F,M', [(1, 1, 4), (5, 2, 4), (64, 500, 32), (300, 3000, 64), (300, 3000, 2)])
def test_random_meshes_vs_double_oracle_bit_exact(Q, F, M):
    """The grid of test_gpu_measure.py::test_mmi_op_random_meshes in float64, plus M = 2 where queries overflow."""
    rng = np.random.RandomState(Q * 1000 + F + 7)
    B = 3

    def soup(n, size):
        return rng.uniform(-1, 1, (B, n, 1, 3)) + rng.normal(0, size, (B, n, 3, 3))
    n_hits, n_over = assert_matches_oracle(soup(Q, 0.15), soup(F, 0.1), M)
    if F >= 500:
        assert n_hits > 0
    if M == 2:
        assert n_over > 0


def test_outputs_and_empty_slots():
    query, target, M = soup_inputs_f64()
    f, b = run(query, target, M)
    B, Q = query.shape[:2]
    assert f.shape == (B, Q * M) and b.shape == (B, Q * M, 2, 3)
    empty = f < 0
    assert (f[empty] == -1).all() and (b[empty] == 0).all() and (~empty).any() and empty.any()


@pytest.mark.parametrize('B,Q,F', [(0, 3, 5), (2, 0, 5), (2, 3, 0)])
def test_empty_sizes(B, Q, F):
    from shapy_b200 import ops
    q = torch.zeros(B, Q, 3, 3, dtype=torch.float64, device='cuda')
    t = torch.zeros(B, F, 3, 3, dtype=torch.float64, device='cuda')
    f, b = ops.mesh_to_mesh_forward(q, t, 4)
    assert f.shape == (B, Q * 4) and f.dtype == torch.int64 and b.shape == (B, Q * 4, 2, 3) and b.dtype == torch.float64
    assert (f == -1).all() and (b == 0).all()


@pytest.mark.parametrize('dq,dt', [(torch.float32, torch.float64), (torch.float64, torch.float32),
                                   (torch.float16, torch.float16), (torch.bfloat16, torch.float64)])
def test_refusals_launch_nothing(dq, dt):
    from shapy_b200 import _lib, ops
    L = _lib.lib()
    n0 = L.shapy_launch_count()
    q = torch.zeros(1, 2, 3, 3, dtype=dq, device='cuda')
    t = torch.zeros(1, 4, 3, 3, dtype=dt, device='cuda')
    with pytest.raises(RuntimeError, match='float32 or both float64'):
        ops.mesh_to_mesh_forward(q, t, 8)
    assert L.shapy_launch_count() == n0


def test_too_many_targets_is_unsupported():
    from shapy_b200 import ops
    q = torch.zeros(1, 2, 3, 3, dtype=torch.float64, device='cuda')
    t = torch.zeros(1, 32769, 3, 3, dtype=torch.float64, device='cuda')
    with pytest.raises(RuntimeError, match=r'code -3\).*32769 target triangles exceed the 32768'):
        ops.mesh_to_mesh_forward(q, t, 8)


def test_deterministic_and_batch_independent(golden_dir):
    from shapy_b200 import ops
    query, tris, M = plane_inputs_f64(golden_dir)
    q, t = torch.from_numpy(query).cuda(), torch.from_numpy(tris).cuda()
    f1, b1 = ops.mesh_to_mesh_forward(q, t, M)
    f2, b2 = ops.mesh_to_mesh_forward(q, t, M)
    assert torch.equal(f1, f2) and torch.equal(b1, b2)
    for i in range(q.shape[0]):
        fi, bi = ops.mesh_to_mesh_forward(q[i:i + 1].contiguous(), t[i:i + 1].contiguous(), M)
        assert torch.equal(fi[0], f1[i]) and torch.equal(bi[0], b1[i]), i


def test_cuda_graph_replay():
    from shapy_b200 import ops
    query, target, M = soup_inputs_f64()
    q, t = torch.from_numpy(query).cuda(), torch.from_numpy(target).cuda()
    want_f, want_b = ops.mesh_to_mesh_forward(q, t, M)              # also sizes the workspace before capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            f, b = ops.mesh_to_mesh_forward(q, t, M)
    f.fill_(7)
    b.fill_(7)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(f, want_f) and torch.equal(b, want_b)


def test_module_in_double():
    from shapy_b200 import ops
    from shapy_b200.mesh_mesh_intersection import MeshMeshIntersection
    query, target, M = soup_inputs_f64()
    q, t = torch.from_numpy(query).cuda(), torch.from_numpy(target).cuda()
    f1, b1 = MeshMeshIntersection(max_collisions=M)(q, t)
    f2, b2 = ops.mesh_to_mesh_forward(q, t, M)
    assert b1.dtype == torch.float64 and torch.equal(f1, f2) and torch.equal(b1, b2)
