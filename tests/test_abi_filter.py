"""The read filter's C-ABI (include/dada2b_filter.h): struct layouts match the ctypes mirror, defaults are
filterAndTrim's, and without a GPU every entry point fails loudly instead of falling back to a CPU path."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_filter_struct_layouts_and_defaults():
    from dada2_b200 import build, filter as fl
    build.build()
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_filter.h"
    int main() {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(dada2b_filter_mate_opts), sizeof(dada2b_filter_opts),
             sizeof(dada2b_filter_out), sizeof(dada2b_filter_stage), offsetof(dada2b_filter_mate_opts, rm_lowcomplex),
             offsetof(dada2b_filter_opts, chunk_n), offsetof(dada2b_filter_out, seq_off), offsetof(dada2b_filter_out, kernel_bytes),
             offsetof(dada2b_filter_out, ms_total), offsetof(dada2b_filter_stage, ee), offsetof(dada2b_filter_stage, complexity));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    M, O, U, S = fl.MateOpts, fl.FilterOpts, fl.FilterOut, fl.Stage
    assert got == [ctypes.sizeof(M), ctypes.sizeof(O), ctypes.sizeof(U), ctypes.sizeof(S), M.rm_lowcomplex.offset, O.chunk_n.offset,
                   U.seq_off.offset, U.kernel_bytes.offset, U.ms_total.offset, S.ee.offset, S.complexity.offset]
    assert ctypes.sizeof(S) == fl.STAGE_DTYPE.itemsize and S.complexity.offset == fl.STAGE_DTYPE.fields["complexity"][1]
    o = O()
    fl._lib().dada2b_filter_default_opts(ctypes.byref(o))              # R/filter.R:402-406
    for m in o.mate:
        assert (m.trunc_q, m.trunc_len, m.trim_left, m.trim_right, m.max_len, m.min_len, m.max_n, m.min_q, m.rm_phix) == (2, 0, 0, 0, -1, 20, 0, 0, 1)
        assert m.max_ee == math.inf and m.rm_lowcomplex == 0.0
    assert o.chunk_n == 100000 and not o.orient_fwd and not o.phix


def test_filter_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dada2_b200 import Dada2bError, filter as fl
    with pytest.raises(Dada2bError, match="no CUDA device"):
        fl.filter_reads(["ACGT" * 10], [np.full(40, 30, np.uint8)], rm_phix=False)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        fl.C_matchRef(["ACGTACGTAC"], "ACGTACGTACGTACGTACGT", 4, True)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        fl.seqComplexity(["ACGTACGTAC"])
    with pytest.raises(Dada2bError, match="no CUDA device"):
        fl.test_filter_stages(["ACGT" * 10], [np.full(40, 30, np.uint8)])


def test_filter_refusals_before_any_device_work():
    from dada2_b200 import Dada2bError, filter as fl
    with pytest.raises(Dada2bError, match="matchIDs"):
        fl.fastqPairedFilter(("a", "b"), ("c", "d"), matchIDs=True)
    with pytest.raises(Dada2bError, match="multithread"):
        fl.filterAndTrim("a", "b", multithread=True)
    with pytest.raises(Dada2bError, match="Phred\\+33"):
        fl.filterAndTrim("a", "b", qualityType="SFastqQuality")
    with pytest.raises(Dada2bError, match="window"):
        fl.seqComplexity(["ACGT"], window=3)
