"""The primer-removal C-ABI (include/dada2b_primer.h): struct layouts match the ctypes mirror, defaults are
removePrimers', and without a GPU every entry point fails loudly instead of falling back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_primer_struct_layouts_and_defaults():
    from dada2_b200 import build, primer as pm
    build.build()
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_primer.h"
    int main() {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %d\n", sizeof(dada2b_primer_opts), sizeof(dada2b_primer_out), sizeof(dada2b_primer_hit),
             offsetof(dada2b_primer_opts, max_mismatch), offsetof(dada2b_primer_opts, orient), offsetof(dada2b_primer_out, reason),
             offsetof(dada2b_primer_out, qual_concat), offsetof(dada2b_primer_out, kernel_bytes), offsetof(dada2b_primer_out, ms_total),
             DADA2B_PRIMER_MAXLEN);
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    O, U, H = pm.PrimerOpts, pm.PrimerOut, pm.Hit
    assert got == [ctypes.sizeof(O), ctypes.sizeof(U), ctypes.sizeof(H), O.max_mismatch.offset, O.orient.offset, U.reason.offset,
                   U.qual_concat.offset, U.kernel_bytes.offset, U.ms_total.offset, pm.MAXLEN]
    assert ctypes.sizeof(H) == pm.HIT_DTYPE.itemsize
    o = O()
    pm._lib().dada2b_primer_default_opts(ctypes.byref(o))              # R/filter.R:81-85
    assert (o.max_mismatch, o.allow_indels, o.trim_fwd, o.trim_rev, o.orient) == (2, 0, 1, 1, 1)
    assert not o.primer_fwd and not o.primer_rev


def test_primer_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dada2_b200 import Dada2bError, primer as pm
    with pytest.raises(Dada2bError, match="no CUDA device"):
        pm.remove_primers_reads(["ACGT" * 10], [np.full(40, 30, np.uint8)], "ACGT")
    with pytest.raises(Dada2bError, match="no CUDA device"):
        pm.test_primer_hits(["ACGT" * 10], [np.full(40, 30, np.uint8)], "ACGT")


def test_primer_refusals_before_any_device_work():
    from dada2_b200 import Dada2bError, primer as pm
    q = [np.full(40, 30, np.uint8)]
    with pytest.raises(Dada2bError, match="allow.indels"):
        pm.removePrimers("a", "b", "ACGT", allow_indels=True)
    with pytest.raises(Dada2bError, match="corresponding output"):
        pm.removePrimers(["a", "b"], ["c"], "ACGT")
    with pytest.raises(Dada2bError, match="base R strings"):
        pm.remove_primers_reads(["ACGT" * 10], q, b"ACGT")
    for kw, msg in ((dict(primer_fwd=""), "empty"), (dict(primer_fwd="A" * 65), "longer than 64"), (dict(primer_fwd="acgt"), "IUPAC"),
                    (dict(primer_fwd="ACGT", max_mismatch=-1), "max.mismatch"), (dict(primer_fwd="ACGT", allow_indels=True), "allow.indels")):
        with pytest.raises(Dada2bError, match=msg):
            pm.remove_primers_reads(["ACGT" * 10], q, **kw)
