"""TEST INFRASTRUCTURE — build recipe for the checkers under oracle/.

* ``build_oracle()``  gcc → oracle/liboracle.so   (the C restatement, oracle/raster_oracle.c)
* ``build_ref()``     nvcc → oracle/_ref/libref_{chn,rgbd,chn_cN}.so — the UNMODIFIED
  reference CUDA library compiled from the sources where they lie under
  /root/reference/submodules/*/cuda_rasterizer (+ our C-ABI shim oracle/ref_shim.cu).
  The reference's own build system (setup.py / CMake) is not run.  The only deviations:
    - ``-include cstdint`` (rasterizer_impl.h:24,40-61 use std::uintptr_t/uint32_t without
      the header; GCC 13 rejects that) — a command-line flag, no source change;
    - the ``chn_cN`` variants need ``#define NUM_CHANNELS N`` (config.h:15) because the
      shipped channel backward is compile-time 3-channel.  config.h is
      included with quotes so it cannot be shadowed from the command line; the recipe
      therefore copies the three .cu/.h files to a temporary directory OUTSIDE the repo,
      rewrites that one line there, compiles, and deletes the copy.  Nothing from the
      reference is ever written into the repository; outputs go only to oracle/_ref/.
  Where the reference sources are absent, prebuilt .so files (git-ignored) are used as they are.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = "/root/reference/submodules"
REF_OUT = os.path.join(HERE, "_ref")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CHN_BWD_VARIANTS = (100, 256, 512)   # libref_chn_c100.so, libref_chn_c256.so, libref_chn_c512.so (K4)


def _newer(target: str, sources) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources if os.path.exists(s))


def _run(cmd, **kw):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + "\n")
        raise RuntimeError(f"build failed: {cmd[0]} (exit {r.returncode})")
    return r.stdout


def build_oracle(verbose: bool = False) -> str:
    src = os.path.join(HERE, "raster_oracle.c")
    out = os.path.join(HERE, "liboracle.so")
    if _newer(out, [src]):
        return out
    # -ffp-contract=off: every fused multiply-add in the restatement is an explicit fmaf()
    # that mirrors the contraction nvcc applies to the reference source (see the file header).
    cmd = ["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math",
           "-fopenmp", "-o", out, src, "-lm"]
    if os.uname().machine == "x86_64":
        cmd.insert(1, "-mfma")
    _run(cmd)
    if verbose:
        print("built", out)
    return out


def _ref_sources(sub: str):
    d = os.path.join(REF_ROOT, sub, "cuda_rasterizer")
    return d, [os.path.join(d, f) for f in ("forward.cu", "backward.cu", "rasterizer_impl.cu")]


def _nvcc_ref(srcdir: str, glm: str, out: str, defines=()):
    srcs = [os.path.join(srcdir, f) for f in ("forward.cu", "backward.cu", "rasterizer_impl.cu")]
    cmd = ["nvcc", *ARCH, "-O3", "-std=c++17", "-include", "cstdint", "-w", "-Xcompiler", "-fPIC",
           "-shared", f"-I{srcdir}", f"-I{glm}", *defines, "-o", out,
           os.path.join(HERE, "ref_shim.cu"), *srcs]
    _run(cmd)


def build_ref(verbose: bool = False):
    """Returns the list of libref_*.so present.  Silently keeps prebuilt files when
    the reference sources are absent."""
    os.makedirs(REF_OUT, exist_ok=True)
    have_ref = os.path.isdir(REF_ROOT)
    shim = os.path.join(HERE, "ref_shim.cu")
    jobs = [("chn", "channel-rasterization", None, []),
            ("rgbd", "rgbd-rasterization", None, ["-DREF_RGBD"])]
    jobs += [(f"chn_c{n}", "channel-rasterization", n, []) for n in CHN_BWD_VARIANTS]
    built = []
    for name, sub, nch, defs in jobs:
        out = os.path.join(REF_OUT, f"libref_{name}.so")
        if not have_ref:
            if os.path.exists(out):
                built.append(out)
            continue
        srcdir, srcs = _ref_sources(sub)
        glm = os.path.join(REF_ROOT, sub, "third_party", "glm")
        if _newer(out, srcs + [shim, os.path.abspath(__file__)]):
            built.append(out)
            continue
        if nch is None:
            _nvcc_ref(srcdir, glm, out, defs)
        else:
            tmp = tempfile.mkdtemp(prefix="sgb200_refbuild_")
            try:
                for f in os.listdir(srcdir):
                    shutil.copy(os.path.join(srcdir, f), os.path.join(tmp, f))
                cfg = os.path.join(tmp, "config.h")
                txt = open(cfg).read()
                if "#define NUM_CHANNELS 3" not in txt:
                    raise RuntimeError("reference config.h changed: NUM_CHANNELS line not found")
                open(cfg, "w").write(txt.replace("#define NUM_CHANNELS 3", f"#define NUM_CHANNELS {nch}"))
                _nvcc_ref(tmp, glm, out, defs)
            finally:
                shutil.rmtree(tmp, ignore_errors=True)
        if verbose:
            print("built", out)
        built.append(out)
    return built


def build_ref_knn(verbose: bool = False):
    """oracle/_ref/libref_knn.so: the unmodified reference simple_knn.cu + oracle/knn_shim.cu."""
    os.makedirs(REF_OUT, exist_ok=True)
    out = os.path.join(REF_OUT, "libref_knn.so")
    srcdir = os.path.join(REF_ROOT, "simple-knn")
    if not os.path.isdir(srcdir):
        return out if os.path.exists(out) else None
    src = os.path.join(srcdir, "simple_knn.cu")
    shim = os.path.join(HERE, "knn_shim.cu")
    if _newer(out, [src, shim, os.path.abspath(__file__)]):
        return out
    # -include cfloat: simple_knn.cu uses FLT_MAX without the header (same class of omission as cstdint above)
    _run(["nvcc", *ARCH, "-O3", "-std=c++17", "-w", "-include", "cfloat", "-Xcompiler", "-fPIC", "-shared",
          f"-I{srcdir}", "-o", out, shim, src])
    if verbose:
        print("built", out)
    return out


if __name__ == "__main__":
    build_oracle(verbose=True)
    print("\n".join(build_ref(verbose=True)))
    print(build_ref_knn(verbose=True))
