"""Builds dada2_b200/libdada2b.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdada2b.so")
SOURCES = ["dd_kernels.cu", "dd_final.cu", "dd_nwfwd.cu", "dd_nwrow.cu", "dd_nwlane.cu", "dd_prescreen.cu", "dd_round.cu", "dd_round2.cu", "dd_driver.cu", "dd_bimera.cu", "dd_bimfwd.cu", "dd_bimfwd16.cu", "dd_merge.cu", "dd_pairs.cu", "dd_derep.cu", "dd_collapse.cu", "dd_align.cu", "dd_filter.cu", "dd_primer.cu", "dd_pool.cu", "dd_taxonomy.cu", "dd_species.cu", "dd_qprofile.cu"]
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
         "-Xcompiler", "-fPIC,-O2,-pthread", "-diag-suppress", "550"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(HERE), "include", f) for f in ("dada2b.h", "dada2b_test.h", "dada2b_bimera.h", "dada2b_merge.h", "dada2b_derep.h", "dada2b_collapse.h", "dada2b_align.h", "dada2b_filter.h", "dada2b_primer.h", "dada2b_pool.h", "dada2b_taxonomy.h", "dada2b_species.h", "dada2b_qprofile.h")]
    deps.append(os.path.abspath(__file__))          # FLAGS (target architecture) live here: a library built with other flags is stale
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for cmd, p in procs:
        out = p.communicate()[0].decode()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-lcudart"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
