"""The sequence-table merge's C-ABI (include/dada2b_seqtab.h): the struct layouts match the ctypes mirror, every
refusal that needs no device is made on the host, and without a GPU the entry point fails loudly instead of falling
back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import seqtab_merge_cases as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_seqtab_merge_struct_layouts():
    from dada2_b200 import build, seqtab
    build.build()
    fi, fo = [f[0] for f in seqtab.SeqtabMergeIn._fields_], [f[0] for f in seqtab.SeqtabMergeOut._fields_]
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_seqtab.h"
    int main() {
      printf("%zu %zu %d %d %d", sizeof(dada2b_seqtab_merge_in), sizeof(dada2b_seqtab_merge_out), DADA2B_ORDER_NONE,
             DADA2B_ORDER_ABUNDANCE, DADA2B_ORDER_NSAMPLES);
    ''' + "".join('printf(" %%zu", offsetof(dada2b_seqtab_merge_in, %s));\n' % f for f in fi) + \
        "".join('printf(" %%zu", offsetof(dada2b_seqtab_merge_out, %s));\n' % f for f in fo) + r'''
      printf("\n");
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    I, O = seqtab.SeqtabMergeIn, seqtab.SeqtabMergeOut
    assert got == [ctypes.sizeof(I), ctypes.sizeof(O), 0, seqtab.ORDER_BY["abundance"], seqtab.ORDER_BY["nsamples"]] + \
        [getattr(I, f).offset for f in fi] + [getattr(O, f).offset for f in fo]


def test_seqtab_merge_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import dada2_b200
    from dada2_b200 import Dada2bError, seqtab
    with pytest.raises(Dada2bError, match="no CUDA device"):
        dada2_b200.mergeSequenceTables(G.t([[1]], [G.S1], "a"), G.t([[2]], [G.S3], "b"), tryRC=True)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        seqtab.merge_columns([np.ones((1, 1), np.int32)] * 2, [[G.S1], [G.S1]], [0, 0], 1)


def test_seqtab_merge_refusals_before_any_device_work():
    G.check_refusals()


def test_seqtab_merge_restatement_colmajor_forms_agree():
    """The restatement's two forms of R's sub-assignment (cell by cell in column-major order, and the last row and
    column of every name) write the same cells."""
    from tests import seqtab_merge_ref as R
    rng = np.random.default_rng(5)
    for _ in range(20):
        ri = rng.integers(0, 6, 150)
        ci = rng.integers(0, 40, 150)
        new = rng.integers(0, 100, (150, 150))
        a = np.zeros((6, 40), np.int64)
        for j in range(len(ci)):
            for i in range(len(ri)):
                a[ri[i], ci[j]] = new[i, j]
        b = np.zeros((6, 40), np.int64)
        R.assign_colmajor(b, ri, ci, new)
        assert np.array_equal(a, b)
