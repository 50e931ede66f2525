"""Build the sm_90a (H100) shared library in-tree, next to the package that loads it.

    python -m vampnet_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The output is vampnet_b200/libvampnet_b200.so (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libvampnet_b200.so")
SOURCES = ["api.cu", "gemm_wgmma.cu", "attention_wgmma.cu", "elementwise.cu", "sampler.cu", "codec.cu", "conv_wgmma.cu", "lora.cu", "onset.cu", "beat.cu", "pitch.cu", "validate.cu", "mel.cu", "tables.cu", "fad.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "vampnet_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    common = [
        NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
        "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
    ]
    if verbose:
        common += ["-Xptxas", "-v"]
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src) + ".o")
        objs.append(obj)
        procs.append((src, subprocess.Popen(common + ["-c", src, "-o", obj], stdout=subprocess.PIPE,
                                            stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {os.path.basename(src)} ---\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    link = [NVCC, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
