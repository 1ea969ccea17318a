"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, exports every
symbol include/*.h declares, its struct layouts match the ctypes mirror, and -- with no GPU -- it fails
loudly instead of falling back to a CPU path."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from dada2_b200 import build
    build.build()
    from dada2_b200 import api
    return api.lib()


def test_library_exports_every_declared_symbol():
    L = _lib()
    names = set()
    for h in sorted(f for f in os.listdir(os.path.join(ROOT, "include")) if f.endswith(".h")):
        src = open(os.path.join(ROOT, "include", h)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names |= set(re.findall(r"\b(dada2b_[a-z_A-Z0-9]+)\s*\(", src))
    assert {"dada2b_run", "dada2b_free", "dada2b_upload", "dada2b_run_resident", "dada2b_ctx_free",
            "dada2b_default_opts", "dada2b_test_pairs", "dada2b_test_calc_pA", "dada2b_test_screen", "dada2b_test_raw_bounds", "dada2b_test_bound", "dada2b_table_bimera", "dada2b_is_bimera",
            "dada2b_bimera_default_opts", "dada2b_test_bimera_pairs", "dada2b_merge_pairs", "dada2b_merge_free",
            "dada2b_merge_default_opts", "dada2b_derep", "dada2b_derep_free", "dada2b_derep_resident"} <= names
    for n in sorted(names):
        assert hasattr(L, n), "libdada2b.so does not export %s" % n


_CTYPE_OF = {"int32_t": "c_int", "uint32_t": "c_uint", "int64_t": "c_long", "uint64_t": "c_ulong", "double": "c_double"}


def test_test_hook_bindings_match_header():
    """Every stage hook of include/dada2b_test.h is bound in api.lib() with one ctypes argument per C parameter, of the same kind:
    a pointer where the header has one, an integer of the same width and sign, a double.  A parameter added to a hook (njobs_hint
    of dada2b_test_loop_nw, dada2b_test_bound) without its binding would shift every later argument."""
    L = _lib()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dada2b_test.h")).read(), flags=re.S)
    protos = re.findall(r"\bint\s+(dada2b_test_\w+)\s*\(([^)]*)\)\s*;", src)
    assert {n for n, _ in protos} >= {"dada2b_test_pairs", "dada2b_test_loop_nw", "dada2b_test_bound", "dada2b_test_raw_bounds"}
    for name, params in protos:
        params = [" ".join(p.split()) for p in params.split(",")]
        argt = getattr(L, name).argtypes
        assert argt is not None and len(argt) == len(params), (name, len(params), argt and len(argt))
        for p, t in zip(params, argt):
            if "*" in p or "[" in p:
                assert t is ctypes.c_void_p or t is ctypes.c_char_p or hasattr(t, "contents"), (name, p, t)
            else:
                ct = p.replace("const ", "").split()[0]
                assert t.__name__ == _CTYPE_OF[ct] or ctypes.sizeof(t) == ctypes.sizeof(getattr(ctypes, _CTYPE_OF[ct])) and \
                    (t.__name__.startswith("c_u") == _CTYPE_OF[ct].startswith("c_u")), (name, p, t)


def test_struct_layouts_match_ctypes_mirror():
    from dada2_b200 import _abi
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b.h"
    int main() {
      printf("%zu %zu %zu %zu %zu %zu\n", sizeof(dada2b_in), sizeof(dada2b_opts), sizeof(dada2b_out),
             offsetof(dada2b_out, subqual_ncol), offsetof(dada2b_out, n_align), offsetof(dada2b_out, ms_device));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = [ctypes.sizeof(_abi.In), ctypes.sizeof(_abi.Opts), ctypes.sizeof(_abi.Out),
            _abi.Out.subqual_ncol.offset, _abi.Out.n_align.offset, _abi.Out.ms_device.offset]
    assert got == want


def test_bimera_struct_layouts_and_defaults():
    from dada2_b200 import bimera
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_bimera.h"
    int main() {
      printf("%zu %zu %zu %zu %zu\n", sizeof(dada2b_bimera_opts), sizeof(dada2b_bimera_stats), offsetof(dada2b_bimera_opts, max_shift),
             offsetof(dada2b_bimera_opts, shard_world), offsetof(dada2b_bimera_stats, ms_k_align));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [ctypes.sizeof(bimera.BimeraOpts), ctypes.sizeof(bimera.BimeraStats), bimera.BimeraOpts.max_shift.offset,
                   bimera.BimeraOpts.shard_world.offset, bimera.BimeraStats.ms_k_align.offset]
    _lib()
    o = bimera._opts()                                          # R/chimeras.R:220, R/dada.R:1-26
    assert (o.min_fold, o.min_abund, o.allow_one_off, o.min_one_off_par_dist, o.match, o.mismatch, o.gap_p, o.max_shift,
            o.shard_rank, o.shard_world) == (1.5, 2, 0, 4, 5, -4, -8, 16, 0, 1)


def test_merge_struct_layouts_and_defaults():
    from dada2_b200 import merge
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_merge.h"
    int main() {
      printf("%zu %zu %zu %zu %zu\n", sizeof(dada2b_merge_opts), sizeof(dada2b_merge_out), offsetof(dada2b_merge_out, cons_off),
             offsetof(dada2b_merge_out, n_cells), offsetof(dada2b_merge_out, ms_total));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [ctypes.sizeof(merge.MergeOpts), ctypes.sizeof(merge.MergeOut), merge.MergeOut.cons_off.offset,
                   merge.MergeOut.n_cells.offset, merge.MergeOut.ms_total.offset]
    o = merge.MergeOpts()
    merge._lib().dada2b_merge_default_opts(ctypes.byref(o))      # R/paired.R:153-155, nwalign(band=-1)
    assert (o.match, o.mismatch, o.gap_p, o.homo_gap_p, o.band, o.trim_overhang) == (1, -64, -64, -64, -1, 0)


def test_derep_struct_layouts():
    from dada2_b200 import derep
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dada2b_derep.h"
    int main() {
      printf("%zu %zu %zu %zu %zu\n", sizeof(dada2b_derep_in), sizeof(dada2b_derep_out), offsetof(dada2b_derep_in, chunk_n),
             offsetof(dada2b_derep_out, map), offsetof(dada2b_derep_out, ms_total));
      return 0;
    }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [ctypes.sizeof(derep.DerepIn), ctypes.sizeof(derep.DerepOut), derep.DerepIn.chunk_n.offset, derep.DerepOut.map.offset,
                   derep.DerepOut.ms_total.offset]


def test_default_opts_are_the_reference_defaults():
    from dada2_b200 import _abi
    L = _lib()
    o = _abi.Opts()
    L.dada2b_default_opts(ctypes.byref(o))
    d = _abi.DEFAULT_OPTS                                       # R/dada.R:1-26
    for k, _t in _abi.Opts._fields_:
        assert getattr(o, k) == (float(d[k]) if _t is ctypes.c_double else int(d[k])), k


def test_no_gpu_means_loud_failure_not_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import dada2_b200
    with pytest.raises(dada2_b200.Dada2bError, match="no CUDA device"):
        dada2_b200.dada_uniques(["ACGTACGTAC"], [1], None, np.ones((16, 41)), np.full((1, 10), 30.0))
    with pytest.raises(dada2_b200.Dada2bError, match="no CUDA device"):
        dada2_b200.bimera.C_table_bimera2(np.ones((1, 2), np.int32), ["ACGTACGTAC", "ACGTACGTAA"])
    with pytest.raises(dada2_b200.Dada2bError, match="no CUDA device"):
        dada2_b200.bimera.C_is_bimera("ACGTACGTAC", ["ACGTACGTAA", "ACGTACGTTT"])
    with pytest.raises(dada2_b200.Dada2bError, match="no CUDA device"):
        dada2_b200.merge.merge_align(["ACGTACGTAC", "ACGTACGTAA"], [0], [1], [1])
    with pytest.raises(dada2_b200.Dada2bError, match="no CUDA device"):
        dada2_b200.derep.derep_reads(["ACGTACGTAC"], [np.full(10, 30, np.uint8)])


def test_product_sources_do_not_touch_the_oracle():
    """The product (package + csrc) must never import/link/execute anything under oracle/."""
    bad = []
    for base, _dirs, files in os.walk(os.path.join(ROOT, "dada2_b200")):
        if "build" in base.split(os.sep)[-1:]:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(base, f), errors="ignore").read()
                if re.search(r"(from|import)\s+oracle|oracle/|liboracle|libdada2ref", txt):
                    bad.append(os.path.join(base, f))
    assert not bad, bad
