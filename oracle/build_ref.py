"""Recipe: compile the REFERENCE's own CUDA extension `localattention` for sm_90a, unmodified, from the sources
where they lie under /root/reference (projects/mmdet3d_plugin/models/utils/ops/locatt_ops/{similar.cu,weighting.cu,
localAttention.cpp,kernels.cuh,utils.cuh,localAttention.h}) into the git-ignored oracle/_ref/.

TEST INFRASTRUCTURE ONLY: the built module is the kernel-level oracle and baseline ("the reference GPU kernel to
beat", SURVEY.md 2.2 / 8(c)(iv)) used by tests/test_gpu_locatt_ref.py and bench.py's reference-kernel timing; nothing
under deepinteraction_b200/ or projects/ may import it.  No reference source is copied into this repository: the
sources are read in place, only the compiled localattention.so lands in oracle/_ref/ (which travels to the GPU box
with the gpurun snapshot; /root/reference itself does not).

Same flags as the reference's JIT recipe (locatt_ops/__init__.py:15-26) plus the explicit sm_90a -gencode (the
reference lets torch pick the visible device's arch; there is no GPU in the build container).

    python oracle/build_ref.py            # -> oracle/_ref/localattention.so   (no-op if /root/reference is absent)
"""
import glob
import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = '/root/reference/projects/mmdet3d_plugin/models/utils/ops/locatt_ops'
OUT_DIR = os.path.join(HERE, '_ref')


def built_path():
    c = glob.glob(os.path.join(OUT_DIR, 'localattention*.so'))
    return c[0] if c else None


def build(verbose=False):
    """Returns the path of the built module, or None when the reference sources are not reachable."""
    if built_path():
        return built_path()
    if not os.path.isdir(REF_DIR):
        return None
    os.makedirs(OUT_DIR, exist_ok=True)
    os.environ.setdefault('TORCH_CUDA_ARCH_LIST', '9.0a')
    from torch.utils import cpp_extension
    srcs = [os.path.join(REF_DIR, f) for f in ('similar.cu', 'weighting.cu', 'localAttention.cpp')]
    cpp_extension.load('localattention', sources=srcs, build_directory=OUT_DIR,
                       extra_cuda_cflags=['-DCUDA_HAS_FP16=1', '-D__CUDA_NO_HALF_OPERATORS__',
                                          '-D__CUDA_NO_HALF_CONVERSIONS__', '-D__CUDA_NO_HALF2_OPERATORS__',
                                          '-gencode', 'arch=compute_90a,code=sm_90a'],
                       is_python_module=False, verbose=verbose)
    return built_path()


def load():
    """Import oracle/_ref/localattention.so (a pybind module) -> module, or None when it was never built."""
    p = built_path()
    if p is None:
        return None
    import torch  # noqa: F401  (the extension links against libtorch)
    spec = importlib.util.spec_from_file_location('localattention', p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv))
