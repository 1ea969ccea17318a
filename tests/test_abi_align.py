"""The nwalign / isShiftDenovo C-ABI (include/dada2b_align.h): struct layouts match the ctypes mirror, defaults are the
reference's, and without a GPU every entry point fails loudly instead of falling back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_align_struct_layouts_and_defaults():
    from dada2_b200 import align, bimera, build
    build.build()
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_align.h"
    int main() {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(dada2b_nwalign_opts), sizeof(dada2b_nwalign_stats),
             offsetof(dada2b_nwalign_opts, vec), offsetof(dada2b_nwalign_stats, ms_total), sizeof(dada2b_shift_opts),
             sizeof(dada2b_shift_stats), offsetof(dada2b_shift_opts, gap_p), offsetof(dada2b_shift_stats, ms_device),
             offsetof(dada2b_shift_stats, ms_total));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    O, S, SO, SS = align.NwalignOpts, align.NwalignStats, bimera.ShiftOpts, bimera.ShiftStats
    assert got == [ctypes.sizeof(O), ctypes.sizeof(S), O.vec.offset, S.ms_total.offset, ctypes.sizeof(SO), ctypes.sizeof(SS),
                   SO.gap_p.offset, SS.ms_device.offset, SS.ms_total.offset]
    o = O()
    align._lib().dada2b_nwalign_default_opts(ctypes.byref(o))          # R/misc.R:179, getDadaOpt defaults
    assert (o.match, o.mismatch, o.gap_p, o.homo_gap_p, o.band, o.endsfree, o.vec) == (5, -4, -8, -8, -1, 1, 0)
    so = SO()
    bimera._shift_lib().dada2b_shift_default_opts(ctypes.byref(so))   # R/chimeras.R:384
    assert (so.min_overlap, so.match, so.mismatch, so.gap_p) == (20, 5, -4, -8)


def test_align_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dada2_b200 import Dada2bError, bimera, isShiftDenovo, nwalign, seqtab
    a, b = "ACGTACGTAC" * 3, "CGTACGTACG" * 3
    with pytest.raises(Dada2bError, match="no CUDA device"):
        nwalign(a, b)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        seqtab.nwhamming(a, b)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        isShiftDenovo({a: 5, b: 3})
    with pytest.raises(Dada2bError, match="no CUDA device"):
        bimera.test_shift_pairs([a, b], [1], [0])
