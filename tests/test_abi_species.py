"""The species C-ABI (include/dada2b_species.h): struct layouts match the ctypes mirror, and without a GPU every entry
point fails loudly instead of falling back to a CPU path."""
import ctypes
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_species_struct_layouts():
    from dada2_b200 import build, species as sp
    build.build()
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_species.h"
    int main() {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d\n", sizeof(dada2b_species_seqs), sizeof(dada2b_species_db_info),
             sizeof(dada2b_species_out), offsetof(dada2b_species_seqs, seq_off), offsetof(dada2b_species_db_info, device_bytes),
             offsetof(dada2b_species_db_info, ms_total), offsetof(dada2b_species_out, species_off), offsetof(dada2b_species_out, hit_refs),
             offsetof(dada2b_species_out, scans), offsetof(dada2b_species_out, max_group), offsetof(dada2b_species_out, ms_scan),
             offsetof(dada2b_species_out, ms_total), DADA2B_SPECIES_ANCHOR);
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    S, I, O = sp.SpeciesSeqs, sp.SpeciesDBInfo, sp.SpeciesOut
    assert got == [ctypes.sizeof(S), ctypes.sizeof(I), ctypes.sizeof(O), S.seq_off.offset, I.device_bytes.offset, I.ms_total.offset,
                   O.species_off.offset, O.hit_refs.offset, O.scans.offset, O.max_group.offset, O.ms_scan.offset, O.ms_total.offset, 32]


def test_species_without_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dada2_b200 import Dada2bError, species as sp
    fa = (["r1 Genus species"], ["ACGT" * 10])
    with pytest.raises(Dada2bError, match="no CUDA device"):
        sp.SpeciesDB(fa)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        sp.assignSpecies(["ACGT"], fa)
    with pytest.raises(Dada2bError, match="no CUDA device"):
        sp.addSpecies((None, ["Genus"]), fa, ["ACGT"])
    L = sp._lib()
    out = ctypes.POINTER(sp.SpeciesOut)()
    eb = ctypes.create_string_buffer(sp.ERRLEN)
    assert L.dada2b_species_assign(None, None, 0, 1, 1, ctypes.byref(out), eb) != 0 and not out
    assert L.dada2b_test_species_hits(None, None, 0, ctypes.byref(out), eb) != 0 and not out
    info = sp.SpeciesDBInfo()
    assert L.dada2b_species_db_info_get(None, ctypes.byref(info)) != 0
