"""The GP entry points of gp.cu checked directly against plain fp64 host arithmetic: backward error
of the Cholesky factor, both residuals of the inverse, the exact structure the prediction GEMM
relies on, alpha, the log-determinant and determinism of the fit at every block shape; prediction,
whitening, W^T products, gradients and cross-covariances from the device's own factors; and the
first bad pivot in info.  Shapes, bounds and the code paths each shape reaches: gp_factor_cases.py."""
import pytest

import gp_factor_cases as cases

pytestmark = pytest.mark.gpu


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
