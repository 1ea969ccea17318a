"""removeBimeraDenovo's test reference (tests/removebim_ref.py) on the CPU restatement of chimera.cpp (oracle/port.cpp)
against the goldens generated through it from the reference's own chimera.cpp (oracle/_ref): per-sample flag matrices,
with and without zero-count queries, and pooled flags, for every table and option set."""
import functools

import pytest

from tests import removebim_cases as RC
from tests import removebim_ref as R

port_flags = functools.partial(R.denovo_flags, backend_name="port")


@pytest.mark.parametrize("name", RC.table_names())
def test_port_per_sample_flags_match_goldens(name):
    RC.check_per_sample(name, port_flags)
    RC.check_per_sample(name, port_flags, opt_ids=[0, 4], zero_queries=True)


@pytest.mark.parametrize("name", RC.table_names())
def test_port_pooled_flags_match_goldens(name):
    RC.check_pooled(name, port_flags)


def test_port_per_sample_table_removal():
    """The matrix branch of the restated removeBimeraDenovo on the golden flags: flagged cells zeroed, all-zero columns
    (the original all-zero column of s_edge too) dropped."""
    import numpy as np
    seqs, mat = RC.table("s_edge")
    flags = RC.golden()["s_edge_o0_persample"].astype(bool)
    out, cols = R.remove_table(mat, seqs, "per-sample", flags=flags)
    keep = np.where(flags, 0, mat).sum(axis=0) > 0
    assert not keep[5] and cols == [s for s, k in zip(seqs, keep) if k]
    assert np.array_equal(out, np.where(flags, 0, mat)[:, keep])
