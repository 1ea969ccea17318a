"""The collapseNoMismatch C-ABI (include/dada2b_collapse.h): struct layouts match the ctypes mirror, defaults are the
reference's, and without a GPU both entry points fail loudly instead of falling back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_collapse_struct_layouts_and_defaults():
    from dada2_b200 import build, seqtab
    build.build()
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_collapse.h"
    int main() {
      printf("%zu %zu %zu %zu %zu\n", sizeof(dada2b_collapse_opts), sizeof(dada2b_collapse_stats), offsetof(dada2b_collapse_opts, vec),
             offsetof(dada2b_collapse_stats, ms_device), offsetof(dada2b_collapse_stats, ms_total));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    S, O = seqtab.CollapseStats, seqtab.CollapseOpts
    assert got == [ctypes.sizeof(O), ctypes.sizeof(S), O.vec.offset, S.ms_device.offset, S.ms_total.offset]
    o = O()
    seqtab._lib().dada2b_collapse_default_opts(ctypes.byref(o))        # R/multiSample.R:104, getDadaOpt defaults
    assert (o.min_overlap, o.match, o.mismatch, o.gap_p, o.band, o.vec) == (20, 5, -4, -8, -1, 1)


def test_collapse_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dada2_b200 import Dada2bError, seqtab
    with pytest.raises(Dada2bError, match="no CUDA device"):
        seqtab.collapse_reps(["ACGTACGTAC", "CGTACGTACG"])
    with pytest.raises(Dada2bError, match="no CUDA device"):
        seqtab.nwhamming("ACGTACGTAC", "CGTACGTACG")
