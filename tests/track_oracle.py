"""The angle tracker of include/music_b200.h (music_b200_set_tracking and the *_tracks entries), restated literally in
fp64: per window predict, measurements, distances, global-nearest-neighbour assignment (scipy's linear_sum_assignment
on the (rows + measurements)-square matrix with dummy costs gate / 2), Joseph-form update, status and initiation.
Feed it the device's own angles, bins (and elevations and CRB) and it returns what the device's tracker must."""
from dataclasses import dataclass
import itertools

import numpy as np
from scipy.optimize import linear_sum_assignment

OFF, FIXED, CRB = 0, 1, 2
EMPTY, TENTATIVE, CONFIRMED = 0, 1, 2
INT_MAX = 2 ** 31 - 1


@dataclass
class Params:
    variance: int = FIXED
    q: float = 0.01
    rate_std0: float = 1.0
    floor_deg: float = 0.5
    crb_scale: float = 1.0
    gate: float = 9.0
    confirm_hits: int = 3
    confirm_window: int = 5
    max_misses: int = 5
    max_tracks: int = 8

    def args(self):
        """the arguments of music_b200_set_tracking after the handle"""
        return (self.variance, self.q, self.rate_std0, self.floor_deg, self.crb_scale, self.gate, self.confirm_hits,
                self.confirm_window, self.max_misses, self.max_tracks)


def wrap360(v):
    return v - 360.0 * np.floor(v / 360.0)


def wrap180(v):
    return v - 360.0 * np.floor((v + 180.0) / 360.0)


def assign(d2, gate):
    """the matched (row, measurement) index pairs of the distance matrix d2 [rows][measurements] (NaN: no distance)"""
    nr, nm = d2.shape
    gated = np.zeros(d2.shape, bool) if d2.size == 0 else np.less_equal(d2, gate, where=~np.isnan(d2), out=np.zeros(d2.shape, bool))
    if not gated.any():
        return []
    N = nr + nm
    C = np.full((N, N), np.inf)
    C[:nr, :nm] = np.where(gated, d2, np.inf)
    C[np.arange(nr), nm + np.arange(nr)] = gate / 2
    C[nr + np.arange(nm), np.arange(nm)] = gate / 2
    C[nr:, nm:] = 0.0
    r, c = linear_sum_assignment(C)
    return sorted((int(t), int(i)) for t, i in zip(r, c) if t < nr and i < nm and gated[t, i])


def assign_brute(d2, gate):
    """every matching of gated pairs enumerated: (the least sum of d2 - gate, its pairs)"""
    nr, nm = d2.shape
    best, best_pairs = 0.0, []
    rows = range(nr)
    for k in range(1, min(nr, nm) + 1):
        for rs in itertools.combinations(rows, k):
            for ms in itertools.permutations(range(nm), k):
                v = [d2[t, i] for t, i in zip(rs, ms)]
                if all(x <= gate for x in v):
                    s = sum(x - gate for x in v)
                    if s < best:
                        best, best_pairs = s, sorted(zip(rs, ms))
    return best, best_pairs


class Tracker:
    """The carry of one handle and the recurrence of one window (step); azel: the (az, el) state."""

    def __init__(self, params, azel=False):
        self.p = params
        self.D = 2 if azel else 1
        self.reset()

    def reset(self):
        T, NS = self.p.max_tracks, 2 * self.D
        self.id = [-1] * T
        self.status = [EMPTY] * T
        self.age, self.hits, self.misses = [0] * T, [0] * T, [0] * T
        self.x = np.zeros((T, NS))
        self.P = np.zeros((T, NS, NS))
        self.next_id = 0

    def _empty(self, t):
        self.id[t], self.status[t], self.age[t], self.hits[t], self.misses[t] = -1, EMPTY, 0, 0, 0
        self.x[t] = 0.0
        self.P[t] = 0.0

    def _measurement(self, ang, el, crb):
        p, D = self.p, self.D
        c2, f2 = p.crb_scale * p.crb_scale, p.floor_deg * p.floor_deg
        z = np.array([float(ang)] if D == 1 else [float(ang), float(el)])
        R = np.zeros((D, D))
        if p.variance == CRB:
            c = np.asarray(crb, np.float64).reshape(-1)
            if not np.all(np.isfinite(c)):
                return None
            if D == 1:
                R[0, 0] = c2 * (c[0] * c[0]) + f2
            else:
                sa, se, rho = c
                R[0, 0] = c2 * (sa * sa) + f2
                R[0, 1] = R[1, 0] = c2 * ((rho * sa) * se)
                R[1, 1] = c2 * (se * se) + f2
        else:
            R[np.arange(D), np.arange(D)] = f2
        return z, R

    def _innovation(self, t, z, R):
        D, x, P = self.D, self.x[t], self.P[t]
        if D == 1:
            nu = np.array([wrap180(z[0] - x[0])])
            S = np.array([[P[0, 0] + R[0, 0]]])
            return nu, S, (nu[0] * nu[0]) / S[0, 0]
        nu = np.array([wrap180(z[0] - x[0]), z[1] - x[2]])
        S00, S01, S11 = P[0, 0] + R[0, 0], P[0, 2] + R[0, 1], P[2, 2] + R[1, 1]
        det = S00 * S11 - S01 * S01
        d2 = ((S11 * nu[0]) * nu[0] - ((2.0 * S01) * nu[0]) * nu[1] + (S00 * nu[1]) * nu[1]) / det
        return nu, np.array([[S00, S01], [S01, S11]]), d2

    def step(self, ang, bins, elev=None, crb=None):
        """one window: (slot_track (n,), track_ids (T,), track_state (T, 3 D) float32)"""
        p, D, NS, T, n = self.p, self.D, 2 * self.D, self.p.max_tracks, len(ang)
        q3, q2 = p.q * (1.0 / 3.0), p.q * 0.5
        # 1. predict
        for t in range(T):
            if self.status[t] == EMPTY:
                continue
            P, x = self.P[t], self.x[t]
            for u in range(D):
                for v in range(D):
                    a, b, c, d = P[2 * u, 2 * v], P[2 * u, 2 * v + 1], P[2 * u + 1, 2 * v], P[2 * u + 1, 2 * v + 1]
                    bd, cd = b + d, c + d
                    a, b, c = (a + c) + bd, bd, cd
                    if u == v:
                        a, b, c, d = a + q3, b + q2, c + q2, d + p.q
                    P[2 * u, 2 * v], P[2 * u, 2 * v + 1], P[2 * u + 1, 2 * v], P[2 * u + 1, 2 * v + 1] = a, b, c, d
            for u in range(D):
                x[2 * u] = x[2 * u] + x[2 * u + 1]
            x[0] = wrap360(x[0])
            self.age[t] = min(self.age[t] + 1, INT_MAX)
        # 2. measurements
        meas = {}
        for i in range(n):
            if bins[i] < 0:
                continue
            m = self._measurement(ang[i], None if elev is None else elev[i], None if crb is None else crb[i])
            if m is not None:
                meas[i] = m
        slots = sorted(meas)
        # 3. distances, 4. assignment
        live = [t for t in range(T) if self.status[t] != EMPTY]
        d2 = np.full((len(live), len(slots)), np.nan)
        for a, t in enumerate(live):
            for b, i in enumerate(slots):
                d2[a, b] = self._innovation(t, *meas[i])[2]
        pairs = [(live[a], slots[b]) for a, b in assign(d2, p.gate)]
        slot_track = np.full(n, -1, np.int32)
        matched_rows = {t for t, _ in pairs}
        matched_slots = {i for _, i in pairs}
        # 5. update
        H = np.zeros((D, NS))
        H[np.arange(D), 2 * np.arange(D)] = 1.0
        for t, i in pairs:
            z, R = meas[i]
            nu, S, _ = self._innovation(t, z, R)
            P, x = self.P[t], self.x[t]
            if D == 1:
                K = P[:, [0]] / S[0, 0]
            else:
                S00, S01, S11 = S[0, 0], S[0, 1], S[1, 1]
                det = S00 * S11 - S01 * S01
                K = np.stack([(P[:, 0] * S11 - P[:, 2] * S01) / det, (P[:, 2] * S00 - P[:, 0] * S01) / det], 1)
            x[:] = x + K @ nu
            x[0] = wrap360(x[0])
            A = np.eye(NS) - K @ H
            Pn = (A @ P) @ A.T + (K @ R) @ K.T
            iu = np.triu_indices(NS)
            P[:] = 0.0
            P[iu] = Pn[iu]
            P[(iu[1], iu[0])] = Pn[iu]
            self.hits[t] = min(self.hits[t] + 1, INT_MAX)
            self.misses[t] = 0
            slot_track[i] = self.id[t]
        for t in live:
            if t not in matched_rows:
                self.misses[t] = min(self.misses[t] + 1, INT_MAX)
        # 6. status
        for t in live:
            if self.status[t] == TENTATIVE:
                if self.hits[t] >= p.confirm_hits:
                    self.status[t] = CONFIRMED
                elif self.hits[t] + (p.confirm_window - self.age[t]) < p.confirm_hits:
                    self._empty(t)
            elif self.misses[t] >= p.max_misses:
                self._empty(t)
        # 7. initiation
        for i in slots:
            if i in matched_slots:
                continue
            free = [t for t in range(T) if self.status[t] == EMPTY]
            if not free:
                continue
            t = free[0]
            z, R = meas[i]
            self.id[t] = self.next_id
            self.next_id = (self.next_id + 1) % 2 ** 31
            self.status[t] = CONFIRMED if p.confirm_hits == 1 else TENTATIVE
            self.age[t], self.hits[t], self.misses[t] = 1, 1, 0
            self.x[t] = 0.0
            self.P[t] = 0.0
            for u in range(D):
                self.x[t, 2 * u] = z[u]
                self.P[t, 2 * u + 1, 2 * u + 1] = p.rate_std0 * p.rate_std0
                for v in range(D):
                    self.P[t, 2 * u, 2 * v] = R[u, v]
            slot_track[i] = self.id[t]
        # 8. outputs
        ids = np.full(T, -1, np.int32)
        state = np.zeros((T, 3 * D), np.float32)
        for t in range(T):
            if self.status[t] != CONFIRMED:
                continue
            ids[t] = self.id[t]
            x, P = self.x[t], self.P[t]
            if D == 1:
                state[t] = [x[0], x[1], np.sqrt(P[0, 0])]
            else:
                state[t] = [x[0], x[1], x[2], x[3], np.sqrt(P[0, 0]), np.sqrt(P[2, 2])]
        return slot_track, ids, state

    def run(self, angles, bins, elev=None, crb=None):
        """every window of angles / bins [W][n] (elev [W][n], crb [W][n] or [W][n][3]) in order: stacked outputs"""
        outs = [self.step(angles[w], bins[w], None if elev is None else elev[w], None if crb is None else crb[w])
                for w in range(len(angles))]
        return tuple(np.stack(o) for o in zip(*outs)) if outs else (None, None, None)

    def snapshot(self):
        """what music_b200_get_tracks returns: rows [T][5] int32, state [T][2D + (2D)^2] fp64, next_id"""
        T, NS = self.p.max_tracks, 2 * self.D
        rows = np.array([[self.id[t], self.status[t], self.age[t], self.hits[t], self.misses[t]] for t in range(T)], np.int32)
        state = np.concatenate([self.x, self.P.reshape(T, NS * NS)], 1)
        return rows, state, self.next_id
