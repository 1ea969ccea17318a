"""The quality profile's C-ABI (include/dada2b_qprofile.h): the struct layout matches the ctypes mirror, and without a GPU
every entry point fails loudly instead of falling back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_qprofile_struct_layout():
    from dada2_b200 import build, qc
    build.build()
    fields = [f[0] for f in qc.QProfileOut._fields_]
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_qprofile.h"
    int main() {
      printf("%zu %d", sizeof(dada2b_qprofile_out), DADA2B_QPROFILE_NSCORE);
    ''' + "".join('printf(" %%zu", offsetof(dada2b_qprofile_out, %s));\n' % f for f in fields) + r'''
      printf("\n");
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    U = qc.QProfileOut
    assert got == [ctypes.sizeof(U), qc.NSCORE] + [getattr(U, f).offset for f in fields]


def test_qprofile_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import dada2_b200
    from dada2_b200 import Dada2bError, qc
    with pytest.raises(Dada2bError, match="no CUDA device"):
        qc.quality_tally(np.array([0, 4], np.int64), np.full(4, 30, np.uint8))
    with pytest.raises(Dada2bError, match="no CUDA device"):
        qc.quality_tally(np.zeros(1, np.int64), np.zeros(0, np.uint8))
    gd = os.path.join(ROOT, "tests", "golden")
    with pytest.raises(Dada2bError, match="no CUDA device"):
        dada2_b200.plotQualityProfile(os.path.join(gd, "sam1F.fastq.gz"))
    with pytest.raises(Dada2bError, match="no CUDA device"):
        dada2_b200.plotComplexity(os.path.join(gd, "sam1F.fastq.gz"), n=10)


def test_qprofile_refusals_before_any_device_work():
    import dada2_b200
    from dada2_b200 import Dada2bError, qc
    gd = os.path.join(ROOT, "tests", "golden")
    with pytest.raises(Dada2bError, match="n must be"):
        dada2_b200.plotQualityProfile(os.path.join(gd, "sam1F.fastq.gz"), n=0)
    with pytest.raises(Dada2bError, match="nosuch"):
        dada2_b200.plotQualityProfile(os.path.join(gd, "nosuch.fastq.gz"))
    with pytest.raises(Dada2bError, match="window"):
        dada2_b200.plotComplexity(os.path.join(gd, "sam1F.fastq.gz"), window=25)
    assert [qc.r_character(v) for v in (500000, 250000, 100000, 1000, 1000000, 1200000)] == \
        ["5e+05", "250000", "1e+05", "1000", "1e+06", "1200000"]
