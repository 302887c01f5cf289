"""shapy_b200 -- H100-native (sm_90a) SHAPY inference hot path behind the reference's own module API.

    from shapy_b200.human_shape.models import build_model      # mirrors human_shape.models
    from shapy_b200 import mesh_mesh_intersect_cuda             # mirrors the reference's CUDA extension
    shapy_b200.install_as_reference()                           # alias both under the reference's names

The compute lives in libshapy_b200.so (C ABI: include/shapy_b200.h), built in-tree by
`python -m shapy_b200.build`.  There is no CPU or PyTorch fallback.
"""
import sys

__version__ = '0.1.0'


def install_as_reference():
    """Registers `human_shape.models` (and sub-packages), `mesh_mesh_intersect_cuda`,
    `mesh_mesh_intersection` and `body_measurements` in sys.modules so that the reference's
    regressor/demo.py and regressor/evaluate.py import the H100 path unchanged."""
    import importlib
    from . import body_measurements, mesh_mesh_intersect_cuda, mesh_mesh_intersection, mesh_mesh_intersection_loss
    models = importlib.import_module('shapy_b200.human_shape.models')
    sys.modules['human_shape.models'] = models
    for sub in ('build', 'backbone', 'backbone.hrnet', 'body_heads', 'body_heads.registry', 'body_models',
                'body_models.body_models', 'body_models.lbs', 'body_models.utils', 'common', 'common.networks',
                'common.pose_utils', 'common.iterative_regressor', 'camera', 'camera.camera_projection'):
        sys.modules[f'human_shape.models.{sub}'] = importlib.import_module(f'shapy_b200.human_shape.models.{sub}')
    if 'human_shape' in sys.modules:
        setattr(sys.modules['human_shape'], 'models', models)
    sys.modules['mesh_mesh_intersect_cuda'] = mesh_mesh_intersect_cuda
    sys.modules['mesh_mesh_intersection'] = mesh_mesh_intersection
    sys.modules['mesh_mesh_intersection.loss'] = mesh_mesh_intersection_loss
    mesh_mesh_intersection.loss = mesh_mesh_intersection_loss
    sys.modules['body_measurements'] = body_measurements
