"""The taxonomy C-ABI (include/dada2b_taxonomy.h): struct layouts match the ctypes mirror, and without a GPU every entry
point fails loudly instead of falling back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_taxonomy_struct_layouts():
    from dada2_b200 import build, taxonomy as tx
    build.build()
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_taxonomy.h"
    int main() {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d %d\n", sizeof(dada2b_tax_opts), sizeof(dada2b_tax_seqs),
             sizeof(dada2b_tax_db_info), sizeof(dada2b_tax_out), offsetof(dada2b_tax_opts, chunk_genera), offsetof(dada2b_tax_seqs, seq_off),
             offsetof(dada2b_tax_db_info, table_bytes), offsetof(dada2b_tax_db_info, ms_total), offsetof(dada2b_tax_out, used_rc),
             offsetof(dada2b_tax_out, kernel_bytes), offsetof(dada2b_tax_out, ms_total), DADA2B_TAX_NBOOT, DADA2B_TAX_MAXKMERS);
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    O, S, I, U = tx.TaxOpts, tx.TaxSeqs, tx.TaxDBInfo, tx.TaxOut
    assert got == [ctypes.sizeof(O), ctypes.sizeof(S), ctypes.sizeof(I), ctypes.sizeof(U), O.chunk_genera.offset, S.seq_off.offset,
                   I.table_bytes.offset, I.ms_total.offset, U.used_rc.offset, U.kernel_bytes.offset, U.ms_total.offset, tx.NBOOT, 9999]
    o = O()
    o.max_table_bytes, o.chunk_genera = 5, 6
    tx._lib().dada2b_tax_default_opts(ctypes.byref(o))
    assert (o.max_table_bytes, o.chunk_genera) == (0, 0)


def test_taxonomy_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dada2_b200 import Dada2bError, taxonomy as tx
    with pytest.raises(Dada2bError, match="no CUDA device"):
        tx.TaxDB.from_arrays(["ACGT" * 10], [1], np.ones((1, 2), np.int32))
    with pytest.raises(Dada2bError, match="no CUDA device"):
        tx.C_assign_taxonomy2(["ACGT" * 20], None, ["ACGT" * 10], [1], np.ones((1, 2), np.int32), False)
