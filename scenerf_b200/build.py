"""Builds libscenerf_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m scenerf_b200.build [--force]

The shared library has a plain C ABI (include/scenerf_b200.h) and links the CUDA runtime statically, so it loads
on a machine without a GPU (symbols can be inspected; any call that touches the device returns SRF_E_CUDA).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.path.join(HERE, "libscenerf_b200.so")
SOURCES = ["api.cu", "ray_kernels.cu", "mlp_simt.cu", "mlp_tc.cu", "pack.cu", "tsdf.cu", "image_ops.cu", "backward.cu", "gemm.cu", "sphere_feature.cu", "gemm_tf32.cu", "preproj.cu", "conv_tf32.cu", "tma.cu", "mesh.cu", "metrics.cu", "color_metrics.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*GENCODE, "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def have_nvcc() -> bool:
    import shutil
    return any(c and (os.path.exists(c) if os.path.isabs(c) else shutil.which(c)) for c in
               (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"))


HASH_PATH = os.path.join(HERE, "build", "source_hash.txt")


def _source_hash() -> str:
    import hashlib
    h = hashlib.sha256()
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(HERE, "..", "include", "scenerf_b200.h")]
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _stale():
    """The library is stale when the CONTENT of csrc/ + the header differs from what it was built from (a hash recorded next to
    the objects) -- not by modification times, which a copy to another machine does not preserve."""
    if not os.path.exists(LIB_PATH) or not os.path.exists(HASH_PATH):
        return True
    with open(HASH_PATH) as f:
        return f.read().strip() != _source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB_PATH
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, pr in procs:
        out, _ = pr.communicate()
        log.append("== %s ==\n%s" % (src, out))
        if pr.returncode:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, out))
    cmd = [_nvcc(), "-shared", "-o", LIB_PATH, *objs, *GENCODE]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(os.path.join(HERE, "build", "nvcc.log"), "w") as f:
        f.write("\n".join(log))
    with open(HASH_PATH, "w") as f:
        f.write(_source_hash())
    if verbose:
        print("\n".join(log))
    return LIB_PATH


def build_variant(name: str, defines) -> str:
    """An experimental build next to the product library: csrc/mlp_tc.cu recompiled with extra -D flags, linked with the
    product's other objects into libscenerf_b200_<name>.so (select it with SCENERF_B200_LIB=<path>).  For A/B runs only."""
    build()
    obj = os.path.join(HERE, "build", "mlp_tc_%s.o" % name)
    cmd = [_nvcc(), *[f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")], *defines, "-c", os.path.join(CSRC, "mlp_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        raise RuntimeError("nvcc failed:\n" + r.stdout)
    objs = [obj if s == "mlp_tc.cu" else os.path.join(HERE, "build", s.replace(".cu", ".o")) for s in SOURCES]
    out = os.path.join(HERE, "libscenerf_b200_%s.so" % name)
    r = subprocess.run([_nvcc(), "-shared", "-o", out, *objs, *GENCODE], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        raise RuntimeError("link failed:\n" + r.stdout)
    return out


if __name__ == "__main__":
    if "--variant" in sys.argv:
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], [a for a in sys.argv[i + 2:] if a.startswith("-D")]))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
