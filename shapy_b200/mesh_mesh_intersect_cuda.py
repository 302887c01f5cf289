"""Drop-in for the reference's only native extension module, `mesh_mesh_intersect_cuda`
(mesh-mesh-intersection/src/mesh_mesh_intersect.cpp:59-64):

    mesh_to_mesh_forward(query_triangles, target_triangles, max_collisions=16, print_timings=False)
        -> [collision_faces (B, Q*M) int64, collision_bcs (B, Q*M, 2, 3)]

Triangles are float32 or float64, both the same, as the reference's AT_DISPATCH_FLOATING_TYPES serves them, and
collision_bcs has their dtype.  In float64 the reference still rounds two things to float: its SAT tolerance CMP
(fabsf / FLT_EPSILON) and the projected intervals of the separating-axis test (fminf / fmaxf).  This module does the
same, so it reports the same pairs; AABBs, the ray test and the barycentrics are computed in double.  Mixed dtypes,
float16 and bfloat16 raise RuntimeError, where the reference throws from `data<scalar_t>()` or does not dispatch.

Batched over B in one set of launches on the CURRENT stream, no device synchronisation, errors as
RuntimeError (the reference printf()s and calls exit(0), op.cu:76-86).
"""
from .ops import mesh_to_mesh_forward  # noqa: F401
