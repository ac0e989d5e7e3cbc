"""Distance('mahalanobis', VI=...) on the host MA2 model against the reference's runs, with the C ABI
replaced by the CPU double (tests/mahalanobis_double.py on top of tests/abi_double.py)."""
import pytest

import abi_double
import mahalanobis_cases as cases
import mahalanobis_double


@pytest.fixture(autouse=True)
def _double(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, mahalanobis_double.TABLE)
    return cpu_double


def test_pilot_matches_reference():
    cases.case_pilot()


@pytest.mark.parametrize('run', cases.RUNS)
def test_rejection_matches_reference(run):
    cases.case_rejection(run)
    assert 'elfi_b200_dist_mahalanobis_thr_f64' in abi_double.CALLS


def test_smc_matches_reference():
    cases.case_smc()
