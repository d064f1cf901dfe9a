"""Build recipe for the product library: nvcc -> semantic-gaussians_b200/libsgb200.so (sm_90a).

No torch headers are involved: the library is a plain C-ABI (include/sgb200.h).  The .so is built
in-tree (git-ignored)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsgb200.so")
SOURCES = ["api.cu", "preprocess.cu", "binning.cu", "blend_fwd.cu", "blend_bwd.cu", "weight_pool.cu", "chn_forward.cu", "chn_dfeature.cu", "chn_chain.cu", "geom_bwd.cu", "fusion.cu", "semantic.cu", "decoded_head.cu", "knn.cu", "nearest.cu", "loss.cu", "metric.cu", "feature_loss.cu", "decoder_loss.cu", "voxelize.cu", "elastic.cu", "adam.cu", "sparse_coords.cu", "sparse_conv.cu", "sparse_conv_half.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def source_hash() -> str:
    """sha256 over csrc/* and include/sgb200.h (sorted by name): the identity baked into the library as
    sgb_build_id() and recomputed by bench.py, so a stale prebuilt .so cannot pass for the sources next to it."""
    import hashlib
    h = hashlib.sha256()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))
    files.append(os.path.join(os.path.dirname(HERE), "include", "sgb200.h"))
    for f in files:
        h.update(os.path.basename(f).encode())
        h.update(open(f, "rb").read())
    return h.hexdigest()[:16]


def _deps():
    d = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    d.append(os.path.join(os.path.dirname(HERE), "include", "sgb200.h"))
    d.append(os.path.abspath(__file__))
    return d


def build(verbose: bool = False, force: bool = False, ptxas_verbose: bool = False) -> str:
    if not force and os.path.exists(OUT):
        t = os.path.getmtime(OUT)
        if all(os.path.getmtime(p) <= t for p in _deps()):
            return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = ["nvcc", *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if src == "api.cu":
            cmd.append(f'-DSGB_BUILD_ID="{source_hash()}"')
        if ptxas_verbose:
            cmd += ["-Xptxas", "-v"]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc {src} failed ---\n{out}\n")
        elif verbose or ptxas_verbose:
            sys.stdout.write(f"--- nvcc {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("nvcc failed for libsgb200")
    r = subprocess.run(["nvcc", "-shared", "-o", OUT, *objs, "-lcudart"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed for libsgb200")
    return OUT


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv, ptxas_verbose="-v" in sys.argv))
