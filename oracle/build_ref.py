"""ORACLE - TEST INFRASTRUCTURE ONLY.

Recipe that compiles the UNMODIFIED reference association extension
(/root/reference/extensions: association.cpp + gpu/nmsBase.cu +
gpu/bodyPartConnectorBase.cu) from the sources where they lie into
oracle/_ref/dapalib_ref*.so.  Nothing is copied; the reference's own setup.py is
not run (this is our own recipe: plain nvcc/g++ through torch's cpp_extension
loader, default -fmad=true and no fast-math exactly like the reference's
CUDAExtension with no extra flags, extensions/setup.py:5-13).

gpu/cuda_cal.cu (dead resize kernels, never called from association.cpp) is left
out; it contributes no symbol used by the module.

The product never loads this.  It is used by tests/test_assoc_gpu.py on the GPU
box as the ground-truth for rows B1-B6 of SURVEY.md section 8 (it cannot execute
without a GPU: dapalib.extract unconditionally launches CUDA kernels,
association.cpp:47-69).

Run:  python oracle/build_ref.py     (only possible where /root/reference exists)
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SMAP_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref")
NAME = "dapalib_ref"


def built_path():
    if not os.path.isdir(OUT):
        return None
    for f in os.listdir(OUT):
        if f.startswith(NAME) and f.endswith(".so"):
            return os.path.join(OUT, f)
    return None


def build(verbose=False):
    ext = os.path.join(REF, "extensions")
    if not os.path.isdir(ext):
        return built_path()
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    from torch.utils.cpp_extension import load

    load(
        name=NAME,
        sources=[
            os.path.join(ext, "association.cpp"),
            os.path.join(ext, "gpu", "nmsBase.cu"),
            os.path.join(ext, "gpu", "bodyPartConnectorBase.cu"),
        ],
        extra_include_paths=[ext],
        build_directory=OUT,
        is_python_module=False,  # do not import here: importing needs no GPU, but keep build() side-effect free
        verbose=verbose,
    )
    return built_path()


def load_ref():
    """Import the built reference module (GPU box only makes sense). Returns module or None."""
    p = built_path()
    if p is None:
        return None
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)

    spec = importlib.util.spec_from_file_location(NAME, p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
