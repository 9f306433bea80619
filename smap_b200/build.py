"""Build libsmap_b200.so (sm_90a only) in-tree with nvcc.  `python -m smap_b200.build [-f]`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libsmap_b200.so")
SOURCES = ["engine.cu", "plan.cu", "assoc.cu", "elementwise.cu", "refine.cu", "preprocess.cu", "jpeg.cu", "png.cu", "jpeg_enc.cu", "png_enc.cu", "overlay.cu", "view3d.cu", "json_out.cpp"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def _newer(a, b):
    return os.path.getmtime(a) > os.path.getmtime(b)


def build_variant(name, defines):
    """A/B variant of the library (tools only): same sources with extra -D flags -> lib/libsmap_b200_<name>.so."""
    os.makedirs(LIBDIR, exist_ok=True)
    objs = []
    for s in SOURCES:
        obj = os.path.join(LIBDIR, "%s_%s.o" % (os.path.splitext(s)[0], name))
        objs.append(obj)
        subprocess.check_call(["nvcc"] + NVCC_FLAGS + ["-D" + d for d in defines] + ["-c", os.path.join(CSRC, s), "-o", obj])
    lib = os.path.join(LIBDIR, "libsmap_b200_%s.so" % name)
    subprocess.check_call(["nvcc", "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return lib


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "smap_b200.h")]
    objs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(LIBDIR, os.path.splitext(s)[0] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or any(_newer(d, obj) for d in deps):
            cmd = ["nvcc"] + NVCC_FLAGS + ["-c", src, "-o", obj]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
                print(" ".join(cmd))
            subprocess.check_call(cmd)
    if force or not os.path.exists(LIB) or any(_newer(o, LIB) for o in objs):
        cmd = ["nvcc", "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    if "--variant" in sys.argv:  # python -m smap_b200.build --variant kymajor SMAPB_TAP_KY_MAJOR
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], sys.argv[i + 2:]))
    else:
        print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
