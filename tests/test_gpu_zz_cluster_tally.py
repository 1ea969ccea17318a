"""The per-cluster tallies and $map of dada()'s output (dd_final.cu: k_cluster_tally) and repeated runs of one resident sample on
the H100.  Cases: tests/cluster_tally_cases.py."""
import pytest

from tests import cluster_tally_cases as C

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", C.GOLDEN_NAMES)
def test_cluster_tally_goldens(name):
    import dada2_b200
    C.run_golden(name, dada2_b200.dada_uniques)


@pytest.mark.parametrize("name", ["many_clusters", "omegaC"])
def test_cluster_tally_samples(name):
    import dada2_b200
    C.run_sample(name, dada2_b200.dada_uniques)


def test_repeated_runs_on_one_context(monkeypatch):
    C.run_repeated(monkeypatch)
