"""Builds libselfrecon_b200.so (the C-ABI product library) with nvcc for sm_90a (H100).

In-tree build: the .so lands in selfreconcode_b200/lib/ (git-ignored).  No torch headers are involved: the library's boundary is plain C
(include/selfrecon_b200.h); torch only supplies device memory and streams on the Python side.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBNAME = "libselfrecon_b200.so"
SOURCES = ["minv3x3.cu", "marching_cubes.cu", "interp2x.cu", "grid_sampler.cu", "mlp_kernels.cu",
           "seg3d.cu", "tc_gemm.cu", "trace_tc.cu", "svals3x3.cu", "tc_wgrad.cu", "raster.cu", "mesh_shade.cu",
           "points_silhouette.cu", "texture_bake.cu", "lbsw_field.cu", "mesh_reg.cu", "frames.cu",
           "normal_net.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.sep not in c or os.path.exists(c)):
            return c
    raise RuntimeError("nvcc not found")


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def lib_path():
    return os.path.join(LIBDIR, LIBNAME)


def build_variant(tag, defines):
    """Tuning helper: builds lib/variants/libselfrecon_b200_<tag>.so with extra -D defines."""
    vdir = os.path.join(LIBDIR, "variants", tag)
    os.makedirs(vdir, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        o = os.path.join(vdir, src.replace(".cu", ".o"))
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + ["-c", os.path.join(CSRC, src), "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    out = os.path.join(LIBDIR, "variants", "libselfrecon_b200_%s.so" % tag)
    subprocess.check_call([nvcc, "-shared", "-o", out] + objs)
    return out


def build(force=False, verbose=True):
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "selfrecon_b200.h"))
    stamp = os.path.join(LIBDIR, ".stamp")
    dig = _digest(deps)
    if not force and os.path.exists(lib_path()) and os.path.exists(stamp):
        if open(stamp).read().strip() == dig:
            return lib_path()
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in srcs:
        o = os.path.join(LIBDIR, os.path.basename(s).replace(".cu", ".o"))
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    cmd = [nvcc, "-shared", "-o", lib_path()] + objs
    if verbose:
        print("[build]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(dig)
    return lib_path()


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
