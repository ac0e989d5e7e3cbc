"""The GP factor checks of gp_factor_cases.py against the CPU test double (LAPACK factors): the
bounds, the exact structure and the first-pivot contract hold for a correct factorisation."""
import pytest

import gp_factor_cases as cases

pytestmark = pytest.mark.usefixtures('cpu_double')


@pytest.mark.parametrize('cond', ['well', 'bad'])
@pytest.mark.parametrize('n,p,ldX', cases.FIT_SMALL)
def test_fit_bounds(n, p, ldX, cond):
    cases.case_fit(n, p, ldX, cond)


@pytest.mark.parametrize('n,p,ldX,cond', cases.FIT_LARGE)
def test_fit_bounds_large(n, p, ldX, cond):
    cases.case_fit(n, p, ldX, cond)


@pytest.mark.parametrize('n,p', cases.PREDICT_N)
def test_predict(n, p):
    cases.case_predict(n, p)


@pytest.mark.parametrize('n,p', cases.WHITEN_N)
def test_whiten_apply_wt(n, p):
    cases.case_whiten_apply_wt(n, p)


@pytest.mark.parametrize('n,p', cases.GRAD_N)
def test_predict_grad(n, p):
    cases.case_predict_grad(n, p)


def test_predict_grad_checks_n_pad():
    cases.case_predict_grad_checks_n_pad()


def test_cross_cov():
    cases.case_cross_cov()


@pytest.mark.parametrize('n,j0,kind', cases.PIVOT_CASES)
def test_first_bad_pivot(n, j0, kind):
    cases.case_first_bad_pivot(n, j0, kind)
