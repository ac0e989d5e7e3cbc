"""elfi_b200_dist_euclid_thr_dev_f64 + elfi_b200_accept_append_f64 on the device: the accepted rows
of several batches, appended without a host round trip, give the reference's best-n bit for bit."""
import pytest

import merge_cases as cases

pytestmark = pytest.mark.gpu


def test_device_thresholds_and_append():
    cases.case_device_thresholds_and_append()


def test_topn_merge_matches_reference_merge():
    cases.case_topn_merge_matches_reference_merge()
