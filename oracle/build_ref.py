"""TEST INFRASTRUCTURE ONLY -- builds the REFERENCE's own BVH operator into oracle/_ref/ (git-ignored, travels to the
GPU box with the snapshot) so the GPU tests can compare shapy_mmi_forward with the real kernel on the same GPU.

Sources are compiled where they lie under /root/reference/mesh-mesh-intersection (never copied into the repo):
    src/mesh_mesh_intersect_cuda_op.cu   (op.cu)       include/*.h(pp)
    src/mesh_mesh_intersect.cpp          (bind.cpp)
op.cu does not compile against torch 2.11 as is: `AT_DISPATCH_FLOATING_TYPES(query_triangles.type(), ...)` at op.cu:996-997
needs `.scalar_type()` (SURVEY.md 8c).  The recipe compiles a scratch copy under /tmp with exactly that one token
changed; nothing else is touched.  Own recipe (nvcc + g++ directly), not the reference's setup.py.

    python oracle/build_ref.py            # ~3 min; no-op when /root/reference is absent or the .so is up to date

The module is named mesh_mesh_intersect_cuda_ref and exports the reference's `mesh_to_mesh_forward`.
"""
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('SHAPY_REFERENCE', '/root/reference')
MMI = os.path.join(REF, 'mesh-mesh-intersection')
OUT_DIR = os.path.join(_HERE, '_ref')
OUT = os.path.join(OUT_DIR, 'mesh_mesh_intersect_cuda_ref.so')
NAME = 'mesh_mesh_intersect_cuda_ref'


def available() -> bool:
    return os.path.isfile(os.path.join(MMI, 'src', 'mesh_mesh_intersect_cuda_op.cu'))


def build(force: bool = False, verbose: bool = False):
    """Returns the path of the built module, or None when the reference tree is not mounted (GPU box: prebuilt file)."""
    if not available():
        return OUT if os.path.exists(OUT) else None
    src_cu = os.path.join(MMI, 'src', 'mesh_mesh_intersect_cuda_op.cu')
    src_cpp = os.path.join(MMI, 'src', 'mesh_mesh_intersect.cpp')
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(src_cu), os.path.getmtime(src_cpp)):
        return OUT
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix='shapy_ref_build_')
    try:
        text = open(src_cu).read()
        old = 'query_triangles.type(), "bvh_tree_building"'
        if text.count(old) != 1:
            raise RuntimeError('build_ref: the dispatch line of op.cu is not where SURVEY.md 8c found it')
        patched = os.path.join(tmp, 'op_patched.cu')
        with open(patched, 'w') as f:
            f.write(text.replace(old, 'query_triangles.scalar_type(), "bvh_tree_building"'))
        inc = [f'-I{p}' for p in ce.include_paths()] + [f'-I{os.path.join(MMI, "include")}', f'-I{sysconfig.get_paths()["include"]}']
        defs = [f'-DTORCH_EXTENSION_NAME={NAME}', '-DTORCH_API_INCLUDE_EXTENSION_H',
                f'-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}']
        nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
        o_cu, o_cpp = os.path.join(tmp, 'op.o'), os.path.join(tmp, 'bind.o')
        run = lambda cmd: subprocess.run(cmd, check=True, capture_output=not verbose)
        run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xcompiler', '-fPIC',
             '--expt-relaxed-constexpr', '--expt-extended-lambda', '-DPRINT_TIMINGS=0', '-DDEBUG_PRINT=0', '-DERROR_CHECKING=1',
             '-DCOLLISION_ORDERING=1', '-w'] + defs + inc +
            ['-c', patched, '-o', o_cu])
        run(['g++', '-O2', '-std=c++17', '-fPIC', '-w'] + defs + inc + ['-c', src_cpp, '-o', o_cpp])
        libs = [f'-L{p}' for p in ce.library_paths()] + [f'-Wl,-rpath,{p}' for p in ce.library_paths()]
        run(['g++', '-shared', '-o', OUT, o_cu, o_cpp] + libs +
            ['-lc10', '-lc10_cuda', '-ltorch_cpu', '-ltorch_cuda', '-ltorch', '-ltorch_python', '-L/usr/local/cuda/lib64', '-lcudart'])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return OUT


def load():
    """Imports the built module (needs a CUDA-capable torch at call time, like the reference's own extension)."""
    import importlib.machinery
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    if not os.path.exists(OUT):
        raise FileNotFoundError(OUT)
    loader = importlib.machinery.ExtensionFileLoader(NAME, OUT)
    spec = importlib.util.spec_from_loader(NAME, loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
