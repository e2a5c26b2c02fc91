"""The tracker's restatement (tests/track_oracle.py) on its own: the assignment against brute-force enumeration, the
confirmation, deletion and id rules at the exact windows, the wrap at 0 / 360 degrees, the filter's consistency (NEES)
on a truth that follows its own model, and two crossing sources keeping their ids."""
import numpy as np
import pytest

import track_oracle as to


def _run(params, angles, bins=None, elev=None, crb=None, azel=False):
    angles = np.asarray(angles, np.float32)
    if angles.ndim == 1:
        angles = angles[:, None]
    bins = np.zeros(angles.shape, np.int32) if bins is None else np.asarray(bins, np.int32)
    tr = to.Tracker(params, azel=azel)
    return tr, tr.run(angles, bins, elev, crb)


@pytest.mark.parametrize("seed", range(40))
def test_assignment_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    nr, nm = rng.integers(1, 6, 2)
    gate = 4.0
    d2 = rng.uniform(0.0, 8.0, (nr, nm))
    d2[rng.random((nr, nm)) < 0.1] = np.nan
    best, pairs = to.assign_brute(d2, gate)
    got = to.assign(d2, gate)
    assert got == pairs, (d2, got, pairs)
    assert np.isclose(sum(d2[t, i] - gate for t, i in got), best)


def test_m_of_n_confirmation_and_deletion():
    p = to.Params(confirm_hits=3, confirm_window=5, max_misses=2, max_tracks=4, floor_deg=0.5, gate=9.0)
    # hit, miss, hit, miss, hit: the third hit comes at age 5 and confirms
    bins = np.array([[0], [-1], [0], [-1], [0], [0]])
    _, (st, ids, _) = _run(p, [50.0] * 6, bins)
    assert list(st[:, 0]) == [0, -1, 0, -1, 0, 0]
    assert list(ids[:, 0]) == [-1, -1, -1, -1, 0, 0]
    # hit, miss, miss, miss: at age 4 hits + (5 - 4) = 2 < 3, deleted there; the next hit starts id 1
    bins = np.array([[0], [-1], [-1], [-1], [0]])
    tr, (st, ids, _) = _run(p, [50.0] * 5, bins)
    assert list(st[:, 0]) == [0, -1, -1, -1, 1]
    rows, _, nxt = tr.snapshot()
    assert rows[0].tolist() == [1, to.TENTATIVE, 1, 1, 0] and nxt == 2


def test_max_misses_deletes_confirmed():
    p = to.Params(confirm_hits=2, confirm_window=2, max_misses=3, max_tracks=2, gate=9.0)
    bins = np.array([[0], [0], [-1], [-1], [-1], [0]])
    _, (st, ids, _) = _run(p, [10.0] * 6, bins)
    assert list(ids[:, 0]) == [-1, 0, 0, 0, -1, -1]
    assert st[5, 0] == 1


def test_ids_only_grow():
    rng = np.random.default_rng(3)
    p = to.Params(confirm_hits=2, confirm_window=3, max_misses=2, max_tracks=4, gate=4.0, floor_deg=1.0)
    ang = rng.uniform(0, 360, (300, 3)).astype(np.float32)
    bins = np.where(rng.random((300, 3)) < 0.7, 0, -1).astype(np.int32)
    tr, (st, ids, _) = _run(p, ang, bins)
    started = [v for w in range(300) for v in st[w] if v >= 0]
    new = []
    seen = set()
    for v in started:
        if v not in seen:
            new.append(v)
            seen.add(v)
    assert new == sorted(new) and new == list(range(len(new)))
    assert tr.next_id == len(new)


def test_full_table_gives_minus_one():
    p = to.Params(max_tracks=2, confirm_hits=1, confirm_window=1, gate=1.0, floor_deg=0.1)
    ang = np.array([[10.0, 100.0, 200.0]], np.float32)
    _, (st, ids, _) = _run(p, ang, np.zeros((1, 3), np.int32))
    assert st[0].tolist() == [0, 1, -1]
    assert ids[0].tolist() == [0, 1]


@pytest.mark.parametrize("azel", [False, True])
def test_wrap_through_zero_is_one_track(azel):
    p = to.Params(confirm_hits=2, confirm_window=3, q=1e-4, floor_deg=0.05, gate=16.0, rate_std0=1.0)
    W = 40
    az = np.mod(359.0 + 0.1 * np.arange(W), 360.0).astype(np.float32)  # 359.9 -> 0.1 between windows 9 and 11
    el = np.full((W, 1), 20.0, np.float32) if azel else None
    _, (st, ids, state) = _run(p, az, elev=el, azel=azel)
    assert np.all(st[:, 0] == 0)
    assert np.all(ids[1:, 0] == 0)
    assert abs(to.wrap180(float(state[-1, 0, 0]) - float(az[-1]))) < 0.05
    assert abs(state[-1, 0, 1] - 0.1) < 0.01


def _nees(azel, seed):
    rng = np.random.default_rng(seed)
    D, W, q, sigma = (2 if azel else 1), 10000, 0.01, 0.5
    F = np.array([[1.0, 1.0], [0.0, 1.0]])
    Qc = q * np.array([[1 / 3, 1 / 2], [1 / 2, 1.0]])
    Lq = np.linalg.cholesky(Qc)
    x = np.array([[180.0, rng.normal()], [10.0, rng.normal()]])[:D]
    truth = np.zeros((W, D, 2))
    for w in range(W):
        if w:
            x = x @ F.T + (Lq @ rng.standard_normal((2, D))).T
        truth[w] = x
    z = truth[..., 0] + sigma * rng.standard_normal((W, D))
    p = to.Params(variance=to.FIXED, q=q, rate_std0=1.0, floor_deg=sigma, gate=1e6, confirm_hits=1, confirm_window=1,
                  max_misses=1, max_tracks=1)
    tr = to.Tracker(p, azel=azel)
    nees = []
    for w in range(W):
        el = None if D == 1 else [z[w, 1]]
        st, _, _ = tr.step([z[w, 0]], [0], el)
        assert st[0] == 0
        e = np.zeros(2 * D)
        for u in range(D):
            e[2 * u] = tr.x[0, 2 * u] - truth[w, u, 0]
            e[2 * u + 1] = tr.x[0, 2 * u + 1] - truth[w, u, 1]
        e[0] = to.wrap180(e[0])
        if w >= 100:
            nees.append(e @ np.linalg.solve(tr.P[0], e))
    return float(np.mean(nees))


@pytest.mark.parametrize("azel,lo,hi", [(False, 1.8, 2.2), (True, 3.6, 4.4)])
def test_filter_consistency_nees(azel, lo, hi):
    m = _nees(azel, 11)
    print("mean NEES", azel, m)
    assert lo <= m <= hi, m


def crossing(W, rates, starts, sigma, rng):
    truth = np.stack([s + r * np.arange(W) for s, r in zip(starts, rates)], 1)
    z = truth + sigma * rng.standard_normal(truth.shape)
    # slots in random order, as slots filled by strength swap between windows
    order = np.argsort(rng.random(truth.shape), 1)
    return truth, np.take_along_axis(z, order, 1), order


def test_crossing_sources_keep_ids():
    rng = np.random.default_rng(5)
    W, sigma = 120, 0.3
    truth, z, order = crossing(W, [0.5, -0.3], [40.0, 80.0], sigma, rng)  # cross near window 50
    p = to.Params(variance=to.FIXED, q=1e-4, rate_std0=1.0, floor_deg=sigma, gate=16.0, confirm_hits=2, confirm_window=3,
                  max_misses=3, max_tracks=4)
    _, (st, ids, state) = _run(p, z)
    src = np.empty_like(st)
    np.put_along_axis(src, order, st, 1)  # src[w][k]: the id that truth k's measurement went to
    before, after = src[5:40], src[60:]
    for k in range(2):
        assert len(set(before[:, k])) == 1 and len(set(after[:, k])) == 1
        assert before[0, k] == after[0, k]
    assert before[0, 0] != before[0, 1]
    assert np.all((ids[5:] >= 0).sum(1) == 2)
