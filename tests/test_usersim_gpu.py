"""User-written CUDA simulators on the device (csrc/usersim.cu, csrc/usersim_rt.cuh).

MA(2) written against the contract reproduces the built-in sim_ma2 kernel bit for bit; its fused
summaries equal the unfused ones and a NumPy fold of the data; rows do not depend on how a batch
is split into launches; a threshold AR(1) with a loop and a data-dependent branch equals sim_ar1
bit for bit when both regimes share one coefficient and follows a NumPy replay of its stream when
they differ; Rejection, SMC and BSL run on a model built with tools.cuda_simulator; compile errors
carry NVRTC's log; the context compiles a (source, shapes, salt) once."""
import numpy as np
import pytest
import torch

import ar1_replay

pytestmark = pytest.mark.gpu

# MA(2): x_k = w_{k+2} + t1 w_{k+1} + t2 w_k, block m giving (w_2m, w_2m+1) and the roundings of
# sim_ma2_kernel; the summaries are the lag-1 and lag-2 autocovariances, each a left fold from 0
MA2_SOURCE = r'''
__device__ void simulate(const double* theta, elfi::RowStream& rng, double* y) {
    const double t1 = theta[0], t2 = theta[1];
    double w0, w1;
    rng.normal2(0, w0, w1);
    for (int k = 0; k < elfi::n_out; k += 2) {
        double a, b;
        rng.normal2(1 + k / 2, a, b);
        y[k] = __dadd_rn(__dadd_rn(a, __dmul_rn(t1, w1)), __dmul_rn(t2, w0));
        if (k + 1 < elfi::n_out)
            y[k + 1] = __dadd_rn(__dadd_rn(b, __dmul_rn(t1, a)), __dmul_rn(t2, w1));
        w0 = a;
        w1 = b;
    }
}

__device__ void summarise(const double* y, double* s) {
    double c1 = 0.0, c2 = 0.0;
    for (int k = 1; k < elfi::n_out; ++k) {
        c1 = __dadd_rn(c1, __dmul_rn(y[k], y[k - 1]));
        if (k >= 2) c2 = __dadd_rn(c2, __dmul_rn(y[k], y[k - 2]));
    }
    s[0] = c1 / (elfi::n_out - 1);
    s[1] = c2 / (elfi::n_out - 2);
}
'''
MA2_SALT = 0x4d413257

# threshold AR(1): x_0 = 0, x_t = phi_1 x_{t-1} + w_t when x_{t-1} > 0, else phi_2 x_{t-1} + w_t;
# w_t is the t-th sequential normal, sim_ar1's convention (block m gives w_2m, w_2m+1)
SETAR_SOURCE = r'''
__device__ void simulate(const double* theta, elfi::RowStream& rng, double* y) {
    double x = 0.0;
    for (int t = 0; t < elfi::n_out; ++t) {
        const double phi = x > 0.0 ? theta[0] : theta[1];
        x = __dadd_rn(__dmul_rn(phi, x), rng.next_normal());
        y[t] = x;
    }
}
'''
AR1_SALT = 0x41523120


def _dev(x):
    from elfi_b200 import device as dev
    return dev.to_device(np.asarray(x, dtype=np.float64))


def _ma2_params(B, seed):
    rs = np.random.RandomState(seed)
    return _dev(rs.uniform(-1.5, 1.5, B)), _dev(rs.uniform(-0.8, 0.8, B))


@pytest.mark.parametrize('n_obs', [2, 50, 100, 1000])
@pytest.mark.parametrize('B,offset', [(1, 7), (1000, 2 ** 32 - 500), (1000000, 12345)])
def test_ma2_reproduces_builtin_kernel(B, offset, n_obs):
    from elfi_b200 import ops
    sim = ops.usersim_compile(MA2_SOURCE, 2, n_obs, salt=MA2_SALT)
    t1, t2 = _ma2_params(B, n_obs)
    key = 2 ** 33 + 17
    Y, S = ops.usersim_run(sim, [t1, t2], seed=key, offset=offset, want_data=True,
                           want_summaries=False)
    assert S is None and Y.shape == (B, n_obs)
    # sim_ma2 takes n_obs >= 3; the first two columns of a row do not depend on n_obs
    X, _ = ops.sim_ma2(t1, t2, max(n_obs, 3), seed=key, offset=offset, want_data=True,
                       want_summaries=False)
    assert torch.equal(Y, X[:, :n_obs])
    assert torch.isfinite(Y).all()


@pytest.mark.parametrize('n_obs', [3, 8, 100, 129, 1000])
def test_fused_summaries_equal_unfused_and_numpy_fold(n_obs):
    from elfi_b200 import ops
    sim = ops.usersim_compile(MA2_SOURCE, 2, n_obs, n_summaries=2, salt=MA2_SALT)
    B = 10007
    t1, t2 = _ma2_params(B, 1)
    _, fused = ops.usersim_run(sim, [t1, t2], seed=99, offset=3)
    Y, unfused = ops.usersim_run(sim, [t1, t2], seed=99, offset=3, want_data=True)
    X = ops.usersim_run(sim, [t1, t2], seed=99, offset=3, want_data=True, want_summaries=False)[0]
    assert torch.equal(Y, X)
    assert torch.equal(fused, unfused)
    assert torch.equal(ops.usersim_summarise(sim, Y), fused)
    y = Y.cpu().numpy()
    fold1 = np.cumsum(y[:, 1:] * y[:, :-1], axis=1)[:, -1] / (n_obs - 1)
    fold2 = np.cumsum(y[:, 2:] * y[:, :-2], axis=1)[:, -1] / (n_obs - 2)
    np.testing.assert_array_equal(fused.cpu().numpy(), np.column_stack([fold1, fold2]))


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 3000])
def test_rows_do_not_depend_on_the_launch(offset):
    from elfi_b200 import ops
    sim = ops.usersim_compile(MA2_SOURCE, 2, 64, n_summaries=2, salt=MA2_SALT)
    B, k = 20000, 6001
    t1, t2 = _ma2_params(B, 2)
    Y, S = ops.usersim_run(sim, [t1, t2], seed=5, offset=offset, want_data=True)
    Ya, Sa = ops.usersim_run(sim, [t1[:k], t2[:k]], seed=5, offset=offset, want_data=True)
    Yb, Sb = ops.usersim_run(sim, [t1[k:], t2[k:]], seed=5, offset=offset + k, want_data=True)
    assert torch.equal(torch.cat([Ya, Yb]), Y)
    assert torch.equal(torch.cat([Sa, Sb]), S)
    _, Fb = ops.usersim_run(sim, [t1[k:], t2[k:]], seed=5, offset=offset + k)
    assert torch.equal(Fb, S[k:])
    # a (batch, p) matrix gives the rows its columns give
    Ym = ops.usersim_run(sim, torch.stack([t1, t2], 1), seed=5, offset=offset, want_data=True)[0]
    assert torch.equal(Ym, Y)


@pytest.mark.parametrize('n_obs', [1, 200, 1001])
def test_setar_equals_sim_ar1_with_one_coefficient(n_obs):
    from elfi_b200 import ops
    sim = ops.usersim_compile(SETAR_SOURCE, 2, n_obs, salt=AR1_SALT)
    B = 30011
    phi = _dev(np.random.RandomState(3).uniform(-1, 1, B))
    Y = ops.usersim_run(sim, [phi, phi], seed=2 ** 40 + 1, offset=77, want_data=True,
                        want_summaries=False)[0]
    X = ops.sim_ar1(phi, n_obs, seed=2 ** 40 + 1, offset=77, want_data=True)[0]
    assert torch.equal(Y, X)


def test_setar_follows_numpy_replay():
    """Distinct regimes: each element within sim_ar1's replay bound, carried through the
    recursion; rows where the replay cannot tell the branch are left out (a few at most)."""
    from elfi_b200 import ops
    B, n_obs, seed, offset = 20000, 150, 2 ** 35 + 3, 2 ** 32 - 100
    sim = ops.usersim_compile(SETAR_SOURCE, 2, n_obs, salt=AR1_SALT)
    rs = np.random.RandomState(4)
    p1, p2 = rs.uniform(-1, 1, B), rs.uniform(-1, 1, B)
    Y = ops.usersim_run(sim, [p1, p2], seed=seed, offset=offset, want_data=True,
                        want_summaries=False)[0].cpu().numpy()
    z, rad = ar1_replay.normals(B, n_obs, seed, offset)
    dz = 1e-14 * np.maximum(1.0, rad)
    eps = 2.0 ** -52
    x, dx = np.zeros(B), np.zeros(B)
    X, err = np.empty((B, n_obs)), np.empty((B, n_obs))
    unsure = np.zeros(B, dtype=bool)
    both_regimes = np.zeros((B, 2), dtype=bool)
    for t in range(n_obs):
        unsure |= (x != 0) & (np.abs(x) <= 4 * dx)
        up = x > 0
        both_regimes[:, 0] |= up
        both_regimes[:, 1] |= ~up
        phi = np.where(up, p1, p2)
        x_new = phi * x + z[:, t]
        dx = np.abs(phi) * dx + dz[:, t] + 2 * eps * (np.abs(phi * x) + np.abs(x_new))
        x = x_new
        X[:, t], err[:, t] = x, 4 * dx
    assert unsure.sum() <= 2, int(unsure.sum())
    assert both_regimes.all(axis=1).mean() > 0.99
    ok = ~unsure
    bad = ~(np.abs(Y[ok] - X[ok]) <= err[ok])
    assert not bad.any(), np.argwhere(bad)[:5]


# ------------------------------------------------------------------------------ end to end
def _user_ma2_model(n_obs=100, seed_obs=4):
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200 import tools
    from elfi_b200.examples import ma2
    sim = tools.cuda_simulator(MA2_SOURCE, 2, n_obs, n_summaries=2, salt=MA2_SALT)
    m = em.ElfiModel()
    em.Prior('uniform', -2, 4, model=m, name='t1')
    em.Prior('uniform', -1, 2, model=m, name='t2')
    em.Simulator(sim, m['t1'], m['t2'], observed=ma2._observed(n_obs, None, seed_obs), name='MA2')
    em.Summary(tools.fused_summary(0, sim), m['MA2'], name='S1')
    em.Summary(tools.fused_summary(1, sim), m['MA2'], name='S2')
    em.Distance('euclidean', m['S1'], m['S2'], name='d')
    dp = elfi.DeviceModelPrior(m)
    return dp.model, dp


def test_rejection_and_smc_on_a_user_simulator():
    """Stock priors and DeviceModelPrior proposals: runs are a function of the seed, and SMC's
    posterior means are those of the built-in kernel on the same model
    (ma2.get_uniform_device_model).  The box prior gives t2 more room below than the reference's
    triangular one, so its posterior mean of t2 lies near 0.15 with either kernel."""
    import elfi_b200 as elfi
    from elfi_b200.examples import ma2
    m, dp = _user_ma2_model()
    runs = [elfi.Rejection(m['d'], batch_size=100000, seed=3).sample(2000, quantile=0.005,
                                                                     bar=False)
            for _ in range(2)]
    assert runs[0].n_sim == 400000
    assert np.array_equal(runs[0].samples_array, runs[1].samples_array)
    quantiles = [0.2, 0.3, 0.3]
    smc = [elfi.SMC(m['d'], batch_size=50000, seed=5, device_proposal=dp).sample(
        5000, quantiles=quantiles, bar=False) for _ in range(2)]
    res = smc[0]
    assert np.array_equal(res.samples_array, smc[1].samples_array)
    thr = [p.threshold for p in res.populations]
    assert thr[0] > thr[1] > thr[2]
    means = res.sample_means_array
    mb, dpb = ma2.get_uniform_device_model(seed_obs=4)
    ref = elfi.SMC(mb['d'], batch_size=50000, seed=5, device_proposal=dpb).sample(
        5000, quantiles=quantiles, bar=False).sample_means_array
    assert np.all(np.abs(means - ref) < 0.03), (means, ref)
    assert abs(means[0] - 0.6) < 0.05 and abs(means[1] - 0.2) < 0.1, means


def test_smc_with_the_reference_priors_passes_the_device_ma2_bar():
    """test_throughput_gpu.py's device-MA2 SMC, its triangular priors and proposals, with the user
    simulator in place of the built-in one."""
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200 import tools
    from elfi_b200.examples import ma2
    sim = tools.cuda_simulator(MA2_SOURCE, 2, 100, n_summaries=2, salt=MA2_SALT)
    m = em.ElfiModel()
    em.Prior(ma2.DevicePrior1, 2, model=m, name='t1')
    em.Prior(ma2.DevicePrior2, m['t1'], 1, name='t2')
    em.Simulator(sim, m['t1'], m['t2'], observed=ma2._observed(100, None, 4), name='MA2')
    em.Summary(tools.fused_summary(0, sim), m['MA2'], name='S1')
    em.Summary(tools.fused_summary(1, sim), m['MA2'], name='S2')
    em.Distance('euclidean', m['S1'], m['S2'], name='d')
    res = elfi.SMC(m['d'], batch_size=50000, seed=5, device_proposal=ma2.DeviceProposal).sample(
        5000, quantiles=[0.2, 0.3, 0.3], bar=False)
    thr = [p.threshold for p in res.populations]
    assert thr[0] > thr[1] > thr[2]
    means = res.sample_means_array
    assert abs(means[0] - 0.6) < 0.05 and abs(means[1] - 0.2) < 0.05, means


def test_observed_summaries_come_from_the_user_kernel():
    from elfi_b200 import device as dev
    from elfi_b200.examples import ma2
    m, _ = _user_ma2_model(n_obs=100, seed_obs=4)
    y = ma2._observed(100, None, 4)
    want = [np.cumsum(y[0, lag:] * y[0, :-lag])[-1] / (100 - lag) for lag in (1, 2)]
    got = [float(np.asarray(dev.to_host(m[s].observed)).ravel()[0]) for s in ('S1', 'S2')]
    assert got == want


def test_bsl_on_a_user_simulator():
    from elfi_b200 import bsl
    m, dp = _user_ma2_model(n_obs=50)
    rs = np.random.RandomState(0)
    params0 = np.column_stack([rs.uniform(.3, .9, 16), rs.uniform(0., .4, 16)])
    sampler = bsl.BSL(m, 500, ['S1', 'S2'], seed=123, device_proposal=dp)
    res = sampler.sample(200, np.array([[.06, .03], [.03, .06]]), params0=params0, burn_in=50,
                         n_chains=16)
    assert res.n_sim == 200 * 16 * 500
    assert 0 < res.acc_rate < 1
    assert np.all(np.isfinite(sampler.state['logposterior']))


# ------------------------------------------------------------------------------ errors, cache
def test_syntax_error_names_the_users_line():
    from elfi_b200 import _lib, ops
    src = ('__device__ void simulate(const double* theta, elfi::RowStream& rng, double* y) {\n'
           '    y[0] = theta[0] + not_declared;\n'
           '}\n')
    before = ops.usersim_compiles()
    with pytest.raises(_lib.ElfiB200Error, match=r'user_source\(2\): error: identifier '
                                                 r'"not_declared" is undefined'):
        ops.usersim_compile(src, 1, 4)
    assert ops.usersim_compiles() == before


def test_missing_functions_raise():
    from elfi_b200 import _lib, ops, tools
    no_sim = '__device__ void summarise(const double* y, double* s) { s[0] = y[0]; }'
    with pytest.raises(_lib.ElfiB200Error, match='must define __device__ void simulate'):
        ops.usersim_compile(no_sim, 1, 4, n_summaries=1)
    no_summ = SETAR_SOURCE
    with pytest.raises(_lib.ElfiB200Error, match='Unresolved extern function'):
        ops.usersim_compile(no_summ, 2, 4, n_summaries=1, salt=AR1_SALT)
    sim = tools.cuda_simulator(no_sim, 1, 4, n_summaries=1)
    with pytest.raises(_lib.ElfiB200Error, match='simulate'):
        sim(np.zeros(3), batch_size=3)


def test_shapes_are_refused_before_nvrtc():
    from elfi_b200 import ops
    before = ops.usersim_compiles()
    for shape in [(17, 4, 0), (2, ops.USERSIM_N_OUT_MAX + 1, 0), (2, 4, ops.USERSIM_N_SUM_MAX + 1)]:
        with pytest.raises(ValueError):
            ops.usersim_compile(MA2_SOURCE, *shape)
    assert ops.usersim_compiles() == before


def test_compile_cache():
    from elfi_b200 import ops
    src = MA2_SOURCE + '\n// cache test\n'
    before = ops.usersim_compiles()
    a = ops.usersim_compile(src, 2, 30, n_summaries=2, salt=11)
    b = ops.usersim_compile(src, 2, 30, n_summaries=2, salt=11)
    assert ops.usersim_compiles() == before + 1
    assert a.handle.value == b.handle.value
    c = ops.usersim_compile(src, 2, 30, n_summaries=2, salt=12)
    assert ops.usersim_compiles() == before + 2
    d = ops.usersim_compile(src, 2, 31, n_summaries=2, salt=11)
    assert ops.usersim_compiles() == before + 3
    # the salt is the stream's: another salt, other data
    t1, t2 = _ma2_params(100, 0)
    ya = ops.usersim_run(a, [t1, t2], seed=1, want_data=True)[0]
    yc = ops.usersim_run(c, [t1, t2], seed=1, want_data=True)[0]
    assert not torch.equal(ya, yc)
    # one release of two references keeps the simulator; the second frees it
    ops.usersim_release(a)
    assert torch.equal(ops.usersim_run(b, [t1, t2], seed=1, want_data=True)[0], ya)
    ops.usersim_release(b)
    with pytest.raises(ValueError, match='released'):
        ops.usersim_run(b, [t1, t2], seed=1)
    e = ops.usersim_compile(src, 2, 30, n_summaries=2, salt=11)
    assert ops.usersim_compiles() == before + 4
    for s in (c, d, e):
        ops.usersim_release(s)
