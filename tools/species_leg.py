"""Measures assignSpecies' native core at Silva scale on one GPU: a synthetic species database of 4*10^5 references
(1 400-1 600 nt, about 6*10^8 nt) resident on the device, searched with 10^4 and 10^5 250-nt queries, 10^4 full-length
queries and a worst case of 10^4 queries sharing their first 64 nt (with the chosen anchors and with every anchor at
offset 0), all with tryRC.  Reports the build (H2D, packing), the scan-and-verify kernel time from device events, the
reduction, the D2H and the hit counts, with the card's name and power limit.  There is no CPU reference arm (the
reference's vcountPDict needs R and Biostrings); the str.find restatement is timed on a few queries and labelled so.
Prints one JSON object."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dada2_b200.species import SpeciesDB  # noqa: E402
from tests import species_ref as S  # noqa: E402
from tests import species_synth as Y  # noqa: E402

KEYS = ("npatterns", "hit_records", "distinct_hits", "scans", "max_group", "gpu_launches", "h2d_bytes", "d2h_bytes", "ms_h2d", "ms_scan",
        "ms_reduce", "ms_d2h", "ms_device", "ms_total")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(db, qs):
    db.raw(qs[:64], True, 1, 0)                                          # warm-up
    t = time.time()
    r = db.raw(qs, True, 1, 0)
    return dict({k: r["stats"][k] for k in KEYS}, wall_s=time.time() - t, queries=len(qs))


def main():
    nref = int(os.environ.get("SPECIES_NREF", 400000))
    res = {"card": card(), "nref": nref}
    t = time.time()
    ids, refs, gseq = Y.database(nref, max(1, nref // 15), seed=41)
    res["gen_s"] = time.time() - t
    t = time.time()
    db = SpeciesDB((ids, refs))
    res["build"] = dict(db.info, wall_s=time.time() - t)
    for nq in (10000, 100000):
        res["short_%d" % nq] = run(db, Y.queries(refs, gseq, nq, seed=42))
    full = Y.queries(refs, gseq, 0, seed=43, full=10000)
    res["full_10000"] = run(db, full)
    worst = Y.shared_prefix(refs, 10000)
    res["shared64_10000"] = run(db, worst)
    os.environ["DADA2B_SPECIES_ANCHOR0"] = "1"
    res["shared64_10000_anchor0"] = run(db, worst)
    del os.environ["DADA2B_SPECIES_ANCHOR0"]
    nsub = int(os.environ.get("SPECIES_RESTATED", 10))
    if nsub:
        R = S.Refs(refs)
        qs = Y.queries(refs, gseq, nsub, seed=42)
        t = time.time()
        R.hits(qs, True)
        res["restatement_str_find"] = {"queries": nsub, "s": time.time() - t, "note": "the tests' Python str.find restatement, not the reference"}
    res["card_after"] = card()
    print(json.dumps(res, default=float))


if __name__ == "__main__":
    main()
