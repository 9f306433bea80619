"""ORACLE - TEST INFRASTRUCTURE ONLY.

Recipe that compiles the UNMODIFIED reference association extension
(/root/reference/extensions: association.cpp + gpu/nmsBase.cu +
gpu/bodyPartConnectorBase.cu) from the sources where they lie into
oracle/_ref/dapalib_ref*.so.  Nothing is copied; the reference's own setup.py is
not run (this is our own recipe: plain nvcc/g++ through torch's cpp_extension
loader, default -fmad=true and no fast-math exactly like the reference's
CUDAExtension with no extra flags, extensions/setup.py:5-13).

A second module, dapalib_ref_dims (oracle/_ref/dims/), is the same three sources
plus our own oracle/ref_map_size.cpp, whose exported ref_set_map_size(h, w) sets
the reference's global heat-map size (association.cpp:21) so that the reference
runs at map sizes other than 128 x 208.  It refuses the sizes at which the
reference's NMS is not deterministic (see that file).  dapalib_ref itself is
built exactly as before, so tests/golden/assoc_ref.npz and its canary keep
meaning what they meant.  The dims module is compiled with -fvisibility=hidden:
its copy of the global cannot interpose with dapalib_ref's in one process.

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
OUT_DIMS = os.path.join(OUT, "dims")
NAME_DIMS = "dapalib_ref_dims"


def built_path(name=NAME, out=OUT):
    if not os.path.isdir(out):
        return None
    for f in os.listdir(out):  # the dims module lives in its own directory, so the two never match each other
        if f.startswith(name) and f.endswith(".so"):
            return os.path.join(out, f)
    return None


def dims_built_path():
    return built_path(NAME_DIMS, OUT_DIMS)


def _sources(ext):
    return [os.path.join(ext, "association.cpp"), os.path.join(ext, "gpu", "nmsBase.cu"),
            os.path.join(ext, "gpu", "bodyPartConnectorBase.cu")]


def build(verbose=False):
    ext = os.path.join(REF, "extensions")
    if not os.path.isdir(ext):
        return built_path()
    os.makedirs(OUT, exist_ok=True)
    os.makedirs(OUT_DIMS, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    from torch.utils.cpp_extension import load

    load(
        name=NAME,
        sources=_sources(ext),
        extra_include_paths=[ext],
        build_directory=OUT,
        is_python_module=False,  # do not import here: importing needs no GPU, but keep build() side-effect free
        verbose=verbose,
    )
    load(
        name=NAME_DIMS,
        sources=_sources(ext) + [os.path.join(HERE, "ref_map_size.cpp")],
        extra_include_paths=[ext],
        extra_cflags=["-fvisibility=hidden"],  # host TUs only: the CUDA sources never see the global
        build_directory=OUT_DIMS,
        is_python_module=False,
        verbose=verbose,
    )
    return built_path()


def _import(name, p):
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)

    spec = importlib.util.spec_from_file_location(name, p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_ref():
    """Import the built reference module (GPU box only makes sense). Returns module or None."""
    p = built_path()
    return None if p is None else _import(NAME, p)


_dims = None


def load_ref_dims():
    """(module, set_map_size) of dapalib_ref_dims, or None when it is not built.  set_map_size(h, w) returns 0, or the
    refusal code of ref_map_size_check (1: smaller than 3 x 3, 2: w % 16 != 0, 3: h * w % 512 != 0), in which case the
    module keeps its size.  The setter is bound through ctypes on the same path, so it reaches the module's own global.
    Importing and setting need no GPU; extract / connect do."""
    global _dims
    if _dims is None:
        p = dims_built_path()
        if p is None:
            return None
        import ctypes

        mod = _import(NAME_DIMS, p)
        lib = ctypes.CDLL(p)
        lib.ref_set_map_size.argtypes = [ctypes.c_int, ctypes.c_int]
        lib.ref_set_map_size.restype = ctypes.c_int
        lib.ref_get_map_size.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
        lib.ref_get_map_size.restype = None

        def set_map_size(h, w):
            return int(lib.ref_set_map_size(int(h), int(w)))

        def get_map_size():
            h, w = ctypes.c_int(), ctypes.c_int()
            lib.ref_get_map_size(ctypes.byref(h), ctypes.byref(w))
            return h.value, w.value

        set_map_size.get = get_map_size
        _dims = (mod, set_map_size)
    return _dims


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv), dims_built_path())
