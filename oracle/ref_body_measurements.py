"""TEST INFRASTRUCTURE ONLY -- the reference's own BodyMeasurements, loaded by path (build container only).

Used by tools/make_golden.py (tests/golden/ref_measure_grad.npz) and by the CPU test that compares
oracle/measure_grad_oracle.py with the live reference; nothing on the GPU box can import it.
"""
import os
import sys
import types

import torch

from oracle.ref_shim import REF, _load

_CACHE = {}
MMI = os.path.join(REF, 'mesh-mesh-intersection')


def available() -> bool:
    return os.path.isfile(os.path.join(MMI, 'body_measurements', 'body_measurements.py'))


def load():
    """The reference's own mesh-mesh-intersection/body_measurements/body_measurements.py, loaded by path, with its
    `mesh_mesh_intersection` import served by the plain-C restatement of the CUDA operator (oracle/mmi_oracle.c), so
    that it runs on the CPU.  Returns (BodyMeasurements class, cfg for the SMPL-X measurement definitions)."""
    if _CACHE:
        return _CACHE['cls'], _CACHE['cfg']
    from loguru import logger
    logger.remove()
    from oracle import measure_oracle

    class MeshMeshIntersection(torch.nn.Module):
        def __init__(self, max_collisions=32):
            super().__init__()
            self.max_collisions = max_collisions

        def forward(self, query_triangles, target_triangles, print_timings=False):
            f, b = measure_oracle.mesh_to_mesh_forward(query_triangles.detach().cpu().numpy(),
                                                       target_triangles.detach().cpu().numpy(), self.max_collisions)
            return torch.from_numpy(f), torch.from_numpy(b)

    stub = types.ModuleType('mesh_mesh_intersection')
    stub.MeshMeshIntersection = MeshMeshIntersection
    saved = sys.modules.get('mesh_mesh_intersection')
    sys.modules['mesh_mesh_intersection'] = stub
    try:
        m = _load('shapy_ref_body_measurements', os.path.join(MMI, 'body_measurements', 'body_measurements.py'))
    finally:
        if saved is None:
            sys.modules.pop('mesh_mesh_intersection', None)
        else:
            sys.modules['mesh_mesh_intersection'] = saved
    cfg = {'meas_definition_path': os.path.join(MMI, 'data', 'measurement_defitions.yaml'),
           'meas_vertices_path': os.path.join(MMI, 'data', 'smplx_measurements.yaml')}
    _CACHE['cls'], _CACHE['cfg'] = m.BodyMeasurements, cfg
    return m.BodyMeasurements, cfg
