"""The row-stream case table against the kernels it is meant to cover, without a GPU: every
reachable registry path has cases on both H100 variants, every consumer, thread-per-row kernel
and row-group instance that distance.cu and summaries.cu launch has a registry entry, and every
registry entry is launched there."""
import os

import numpy as np
import pytest

import rowstream_cases as cases

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'elfi_b200', 'csrc')


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


@pytest.mark.parametrize('config', sorted(cases.CONFIGS))
def test_table_covers_every_path(config):
    sm, optin = cases.CONFIGS[config]
    missing = cases.uncovered(sm, optin)
    assert not missing, '{}: no case reaches {}'.format(config, missing)


@pytest.mark.parametrize('config', sorted(cases.CONFIGS))
def test_every_ring_path_has_a_wrap_case(config):
    sm, optin = cases.CONFIGS[config]
    rings = set()
    wrapped = set()
    for c in cases.table(sm, optin):
        if cases.ring(c, optin) is None:
            continue
        p = cases.primary(c, optin)
        rings.add(p)
        if c.wrap:
            wrapped.add(p)
            w, ns, G = cases.ring(c, optin)
            tiles = -(-c.B // cases.RS_BOX_ROWS)
            assert (tiles // (sm * w)) * G > 2 * ns, c.ident()
    assert rings - wrapped == set()


@pytest.mark.parametrize('config', sorted(cases.CONFIGS))
def test_every_path_gets_every_layout_it_admits(config):
    sm, optin = cases.CONFIGS[config]
    gaps = cases.layout_gaps(cases.table(sm, optin), optin)
    assert not gaps, '{}: (path, layout) admitted but never run: {}'.format(config, gaps)


def test_layout_gaps_are_named(monkeypatch):
    monkeypatch.setattr(cases, 'THRESHOLD_LAYOUTS', ('contig', 'ld_even'))
    gaps = cases.layout_gaps(cases.table(*cases.NOMINAL), cases.NOMINAL[1])
    assert ('meanvar:BoxTree', 'b1') in gaps and ('autocov:Tree<1,2>', 'off2') in gaps


def test_representatives_cover_every_path():
    sm, optin = cases.NOMINAL
    rep = cases.representatives(cases.table(sm, optin), optin)
    assert set(cases.reachable(optin)) <= set(rep)
    assert all(not c.wrap for c in rep.values())


def test_source_scan_finds_only_registered_kernels():
    keys = cases.scan_sources(_read('distance.cu'), _read('summaries.cu'))
    # the scan itself: it must see the typedef'd metric consumer and every row-group instance
    assert 'MetricConsumer' in keys
    assert {'rowgroup<{},{}>'.format(nb, w) for nb in (1, 2, 3, 4) for w in (8, 6)} <= keys
    assert {'dist_direct_kernel', 'metric_direct_kernel', 'seg_direct_kernel',
            'summary_direct_kernel'} <= keys
    missing = sorted(k for k in keys if not cases.registry_has(k))
    assert not missing, 'launched but not in the registry: {}'.format(missing)


def test_source_scan_finds_every_registered_kernel():
    keys = cases.scan_sources(_read('distance.cu'), _read('summaries.cu'))
    # a template name does not stand for another template it is a substring of
    assert not cases.launched(keys, 'AutocovConsumer<1,2>')
    stale = sorted(p.name for p in cases.REGISTRY.values() if not cases.launched(keys, p.consumer))
    assert not stale, 'in the registry but never launched: {}'.format(stale)


def test_source_scan_flags_an_unregistered_consumer():
    text = _read('distance.cu') + '\nrowstream_launch<BrandNewConsumer>(ctx, S, ld, B, D, 0, p, s);\n'
    keys = cases.scan_sources(text, _read('summaries.cu'))
    assert [k for k in keys if not cases.registry_has(k)] == ['BrandNewConsumer']


def test_dropping_a_shape_names_the_uncovered_path(monkeypatch):
    shapes = cases._shapes
    monkeypatch.setattr(cases, '_shapes', lambda optin: [
        s for s in shapes(optin) if not (s[0] == 'meanvar' and s[1]['D'] in (58, 62))])
    assert cases.uncovered(*cases.NOMINAL) == ['meanvar:rowgroup<4,6>']


def test_thresholds_restated():
    """Spot values of the restatement at the H100's 227 KiB opt-in."""
    sm, optin = cases.NOMINAL
    assert cases.rs_pick_stages(optin, 0) == 6
    assert cases._max_streaming_D(optin, 1) == 20720
    assert cases.fused_moments_warps(optin, 2, 368, 2) == 12
    assert cases.fused_moments_warps(optin, 2, 512, 2) == 8
    assert [n for n in range(2, 65, 4) if cases.rowgroup_warps(optin, n) == 6] == [58, 62]
    assert cases.predict(cases.Case(family='meanvar', D=50, ld=50, off=2), optin) == \
        {'meanvar:rowgroup<4,8>'}
    assert cases.predict(cases.Case(family='meanvar', D=50, ld=52, off=0), optin) == \
        {'meanvar:Regs<4>'}
    assert cases.predict(cases.Case(family='autocov', D=100, ld=100, off=0, lags=(1, 2, 3, 7)),
                         optin) == {'autocov:Leaf<1,2>', 'autocov:Leaf<3,-1>', 'summary:direct'}


def test_kernel_name_matching():
    launched = ['void elfi::rowstream_kernel<elfi::AutocovBoxConsumer<elfi::TreeSum<6>, 1, (int)-1>, 8>'
                '(CUtensorMap_st, long, int, int, elfi::SummaryParams)',
                'void elfi::compact_mask_kernel(const unsigned int*, long, long, int*, long*)']
    assert cases.paths_in(launched) == {'autocov:Tree<1,-1>'}
    assert cases.paths_in(['void elfi::rowstream_kernel<elfi::NestedMomentsConsumer<2>, 12>(...)']) \
        == {'mom:NestedMoments<2>/12w'}


def test_longdouble_reference_against_fractions():
    cases.longdouble_reference_is_exact()


def test_moments_checker_rejects_the_unshifted_formula():
    """One pass without the shift on data at an offset of 1e8 misses the bound by orders of
    magnitude; the shifted form summed sequentially (depth B, not h) still stays inside it."""
    x = cases.accuracy_data('offset_1e8')
    B, D = x.shape
    h = cases.colmoments_depth(D, B, cases.NOMINAL[0])
    s1, s2 = np.cumsum(x, axis=0)[-1], np.cumsum(x * x, axis=0)[-1]
    with pytest.raises(AssertionError):
        cases.check_moments(x, s1 / B, s2 - s1 * s1 / B, h, 'unshifted')
    d = x - x[0]
    t1, t2 = np.cumsum(d, axis=0)[-1], np.cumsum(d * d, axis=0)[-1]
    cases.check_moments(x, x[0] + t1 / B, t2 - t1 * t1 / B, h, 'shifted')
