"""Bodies of the tests of the sync-free batch -> candidate-buffer path (shared by the CPU-double
and GPU collections): device-resident thresholds (elfi_b200_dist_euclid_thr_dev_f64), the append
of accepted rows with device-side counts (elfi_b200_accept_append_f64) and the final best-n, all
against the reference's own merge arithmetic (elfi/methods/inference/samplers.py:209-237)."""
import numpy as np

import elfi_oracle as o


def reference_merge(batches, thr, n, pad=np.inf):
    """samplers.py:209-237 restated on the host: mask, copy to the tail, argsort over n + B.

    Each batch maps output names to (B,) or (B, width) arrays; 'd' holds the K distance columns
    and a row is accepted when every column is within its threshold (thr: a scalar or K values).
    The rows are ranked by the LAST distance column, as the reference ranks nested distances.
    The argsort is stable: the project promises that ties keep their append order (merge_topn,
    argsort, CandidateBuffer.best), while the reference's own np.argsort is a quicksort, whose
    order among ties is unspecified.  The distances of the rows not yet filled start at `pad`:
    the reference's +inf, or NaN, which ranks after an accepted +inf distance (the reference
    ranks its padding first among such ties).  Returns the first n rows of every output."""
    B = len(batches[0]['d'])
    state = {k: np.zeros((n + B,) + np.shape(v)[1:]) for k, v in batches[0].items()}
    state['d'][:] = pad
    for b in batches:
        d = np.asarray(b['d']).reshape(B, -1)
        acc = np.all(d <= np.atleast_1d(thr), axis=1)
        k = int(acc.sum())
        if k:
            for name in state:
                state[name][-k:] = b[name][acc]
        order = np.argsort(state['d'].reshape(n + B, -1)[:, -1], kind='stable')
        for name in state:
            state[name][:] = state[name][order]
    return {k: v[:n] for k, v in state.items()}


def case_device_thresholds_and_append():
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(3)
    B, D, n = 5000, 24, 300
    obs = rs.randn(1, D)
    batches_host, batches_S, buf = [], [], ops.CandidateBuffer(n + 2 * B, [1, 1, 1])
    thr = None
    for step in range(4):
        S = rs.randn(B, D)
        t1, t2 = rs.rand(B), rs.rand(B)
        ref_d = o.cdist_euclid(S, obs)
        if thr is None:
            thr = float(np.quantile(ref_d, 0.04))
            thr_dev = dev.to_device(np.array([thr]))
        d, (idx, n_acc) = ops.dist_euclid(S, obs, thresholds=thr_dev, sync=False)
        assert np.array_equal(d.cpu().numpy(), ref_d)
        k = int(n_acc.item())
        assert np.array_equal(idx[:k].cpu().numpy(), o.accept_indices(ref_d, thr))
        buf.append([d, dev.to_device(t1), dev.to_device(t2)], idx, n_acc, B)
        batches_host.append({'d': ref_d, 't1': t1, 't2': t2})
        batches_S.append(S)
    top, count, dropped = buf.best(n)
    want = reference_merge(batches_host, thr, n)
    total = sum(int((b['d'] <= thr).sum()) for b in batches_host)
    assert count == total and dropped == 0
    top = top.cpu().numpy()
    m = min(n, total)
    assert np.array_equal(top[:, 0], want['d'][:m])
    assert np.array_equal(top[:, 1], want['t1'][:m])
    assert np.array_equal(top[:, 2], want['t2'][:m])
    # the same batches through the one-call form (elfi_b200_rejection_batch_f64, arguments bound
    # once): identical candidate buffer
    import torch
    bound = ops.CandidateBuffer(n + 2 * B, [1, 1, 1])
    Sd = dev.to_device(batches_S[0])
    d_out, idx_out = dev.empty((B,)), dev.empty((B,), dtype=torch.int32)
    n_out = dev.zeros((1,), dtype=torch.int64)
    t1d, t2d = dev.to_device(batches_host[0]['t1']), dev.to_device(batches_host[0]['t2'])
    run = bound.bind_batch(Sd, dev.to_device(obs.ravel()), [thr], d_out, idx_out, n_out, [t1d, t2d])
    for S_h, b in zip(batches_S, batches_host):
        Sd.copy_(dev.to_device(S_h))
        t1d.copy_(dev.to_device(b['t1']))
        t2d.copy_(dev.to_device(b['t2']))
        run()
    top2, count2, dropped2 = bound.best(n)
    assert count2 == count and dropped2 == 0
    assert np.array_equal(top2.cpu().numpy(), top)
    # a full buffer drops the overflow and says so
    small = ops.CandidateBuffer(10, [1])
    dd, (idx, n_acc) = ops.dist_euclid(S, obs, thresholds=dev.to_device(np.array([np.inf])),
                                       sync=False)
    small.append([dd], idx, n_acc, B)
    rows, count, dropped = small.best(10)
    assert count == 10 and dropped == B - 10
    assert np.array_equal(np.sort(rows.cpu().numpy()[:, 0]), np.sort(ref_d[:10]))
    # 2-d source (nested distances keep all their columns) and identity indices
    wide = ops.CandidateBuffer(64, [2, 1])
    a = dev.to_device(rs.randn(40, 2))
    bcol = dev.to_device(rs.randn(40))
    cnt = dev.to_device(np.array([40]), dtype=__import__('torch').int64)
    wide.append([a, bcol], None, cnt, 40)
    assert int(wide.count.item()) == 40
    got = wide.rows[:40].cpu().numpy()
    assert np.array_equal(got[:, :2], a.cpu().numpy()) and np.array_equal(got[:, 2], bcol.cpu().numpy())


def case_topn_merge_matches_reference_merge():
    """elfi_b200_topn_merge_f64 (ops.merge_topn) against the reference's append + argsort +
    permute (samplers.py:226-237): several batches, a (rows, K) distance matrix whose LAST column
    is the key, a 1-d and a 2-d payload, ties and a NaN key, the buffer filling up from empty."""
    import torch
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(11)
    n, B, K = 300, 1000, 3
    state = {'d': dev.empty((n, K)), 'p': dev.empty((n,)), 'S': dev.empty((n, 5))}
    host = {'d': np.zeros((0, K)), 'p': np.zeros(0), 'S': np.zeros((0, 5))}
    nv = 0
    for it in range(5):
        d = np.abs(rs.randn(B, K))
        d[::7, -1] = d[3, -1]                      # ties: stable order decides
        if it == 2:
            d[5, -1] = np.nan                       # ranks last
        batch = {'d': d, 'p': rs.randn(B), 'S': rs.randn(B, 5)}
        if it % 2:
            acc = np.nonzero(d[:, -1] <= 0.5)[0].astype(np.int32)
            map_b = dev.to_device(acc, dtype=torch.int32)
        else:
            acc, map_b = np.arange(B), None
        n_out = min(n, nv + len(acc))
        names = list(state)
        bdev = {k: dev.to_device(batch[k]) for k in names}
        tops = ops.merge_topn([state[k][:nv] for k in names], [bdev[k] for k in names],
                              state['d'][:nv, -1], bdev['d'][:, -1], map_b, n_out)
        cat = {k: np.concatenate([host[k], batch[k][acc]]) for k in names}
        order = np.argsort(cat['d'][:, -1], kind='stable')[:n_out]
        for k, top in zip(names, tops):
            want = cat[k][order]
            got = top.cpu().numpy()
            assert got.shape == want.shape and np.array_equal(got, want, equal_nan=True), (it, k)
            host[k] = want
            state[k][:n_out] = top
        nv = n_out
    assert nv == n
    # nothing to keep / nothing to merge
    empty = ops.merge_topn([state['p'][:0]], [dev.to_device(np.zeros(4))], state['d'][:0, -1],
                           dev.to_device(np.ones(4)), None, 0)
    assert empty[0].shape == (0,)
