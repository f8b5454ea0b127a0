"""Host restatement of the counterfactual policy evaluation (reagent/evaluation/), in numpy, with
no reference code: the episode recursions, the DR rows and the weighted-DR j-step statistics in
episode layout.  tests/test_ope_cpu.py pins it to the goldens of oracle/make_ope_golden.py; the
GPU tests and profiles/time_ope.py use it as the host baseline."""
import numpy as np
import scipy.optimize
import scipy.stats

MAGIC_J = 25
SUBSETS = 25
CONF = 0.9


def sort_order(mdp_id, seq):
    mdp_id, seq = np.asarray(mdp_id).reshape(-1), np.asarray(seq).reshape(-1)
    return np.lexsort((np.arange(len(mdp_id)), seq, mdp_id))


def episode_offsets(mdp_id):
    m = np.asarray(mdp_id).reshape(-1)
    starts = np.flatnonzero(np.r_[True, m[1:] != m[:-1]])
    return np.r_[starts, len(m)]


def logged_values(x, mdp_id, seq, gamma):
    """Column 0 recursion in float32 inside each run of equal mdp_id; other columns copied."""
    out = np.array(x, dtype=np.float32, copy=True)
    seq = np.asarray(seq).reshape(-1)
    off = episode_offsets(mdp_id)
    for lo, hi in zip(off[:-1], off[1:]):
        for r in range(hi - 2, lo - 1, -1):
            g = np.float32(gamma ** float(seq[r + 1] - seq[r]))
            out[r, 0] = np.float32(out[r, 0] + np.float32(out[r + 1, 0] * g))
    return out


def _rowdot(a, b):
    """torch.sum(a * b, dim=1) in float32, in torch's CPU order for a short row: k = 8 (A >= 8)
    or 4 (A >= 4) strided accumulators, added in order"""
    A = a.shape[1]
    k = 8 if A >= 8 else (4 if A >= 4 else 1)
    p = (a.astype(np.float32) * b.astype(np.float32)).astype(np.float32)
    s = None
    for j in range(min(k, A)):
        acc = p[:, j].copy()
        for i in range(j + k, A, k):
            acc = (acc + p[:, i]).astype(np.float32)
        s = acc if s is None else (s + acc).astype(np.float32)
    return s


def sdr_episodes(prop, qv, am, r, lp, mdp_id, gamma):
    v, ql = _rowdot(prop, qv), _rowdot(qv, am)
    w = (_rowdot(prop, am) / lp.reshape(-1)).astype(np.float32)
    r = r.reshape(-1).astype(np.float32)
    g = np.float32(gamma)
    off = episode_offsets(mdp_id)
    drs, vals = [], []
    for lo, hi in zip(off[:-1], off[1:]):
        dr = val = np.float32(0)
        for j in range(hi - 1, lo - 1, -1):
            dr = np.float32(v[j] + np.float32(w[j] * np.float32(np.float32(r[j] + np.float32(g * dr)) - ql[j])))
            val = np.float32(np.float32(val * g) + r[j])
        drs.append(dr)
        vals.append(val)
    return np.array(drs, dtype=np.float32), np.array(vals, dtype=np.float32)


def dr_rows(prop, mr, am, r, mrl, lp):
    w = (_rowdot(prop, am) / lp.reshape(-1)).astype(np.float32)
    dm = _rowdot(prop, mr)
    r, mrl = r.reshape(-1), mrl.reshape(-1)
    return dm, (w * r).astype(np.float32), ((w * (r - mrl)).astype(np.float32) + dm).astype(np.float32)


def wsdr_stats(prop, qv, am, r, lp, mdp_id, gamma, num_j_steps):
    """(j_steps, j-step returns, cov, subset infinite-step returns, mean discounted return)
    with the reference's self-normalised weights, in float64 over episode layout."""
    off = episode_offsets(mdp_id)
    E = len(off) - 1
    lens = np.diff(off)
    L = int(lens.max())
    tp = (prop.astype(np.float64) * am).sum(1)
    sv = (prop.astype(np.float64) * qv).sum(1)
    ql = (qv.astype(np.float64) * am).sum(1)
    iw = tp / lp.reshape(-1)
    rr = r.reshape(-1).astype(np.float64)
    traj = np.repeat(np.arange(E), lens)
    step = np.arange(len(rr)) - off[:-1][traj]
    w = np.empty_like(iw)
    for lo, hi in zip(off[:-1], off[1:]):
        w[lo:hi] = np.cumprod(iw[lo:hi])
    disc = gamma ** np.arange(L, dtype=np.float64)

    def returns(members, js_list):
        """[len(js_list), len(members)] j-step returns under weights normalised over `members`."""
        n = len(members)
        inset = np.zeros(E, dtype=bool)
        inset[members] = True
        rows = inset[traj]
        col = np.bincount(step[rows], weights=w[rows], minlength=L)[step]
        wn = np.where(col == 0, 1.0 / n, w / np.where(col == 0, 1.0, col))
        prev = np.where(step == 0, 1.0 / n, np.r_[0.0, wn[:-1]])
        wd, wde = disc[step] * wn, disc[step] * prev
        isr = np.r_[0.0, np.cumsum(np.where(rows, wd * rr, 0.0))]
        cv = np.r_[0.0, np.cumsum(np.where(rows, wd * ql - wde * sv, 0.0))]
        lo, ln = off[members], lens[members]
        out = np.zeros((len(js_list), n))
        for k, js in enumerate(js_list):
            end = lo + np.minimum(js, ln - 1) + 1  # one past the last summed row
            a = np.where(js >= 0, isr[end] - isr[lo], 0.0)
            c = np.where(js >= 0, cv[end] - cv[lo], 0.0)
            nxt = np.minimum(lo + js + 1, len(rr) - 1)
            dm = np.where(js + 1 < ln, wde[nxt] * sv[nxt], 0.0)
            out[k] = a + dm - c
        return out

    j_steps = [float("inf")]
    if num_j_steps > 1:
        j_steps.append(-1)
    if num_j_steps > 2:
        interval = L // (num_j_steps - 1)
        j_steps += [i * interval for i in range(1, num_j_steps - 1)]
    js_list = [int(min(j, L - 1)) for j in j_steps]
    ret = returns(np.arange(E), js_list)
    cov = np.cov(ret) if len(j_steps) > 1 else None
    subsets = []
    if len(j_steps) > 1:
        S = int(min(E / 2, SUBSETS))
        interval = E / S
        for i in range(S):
            members = np.arange(int(i * interval), int((i + 1) * interval))
            subsets.append(returns(members, [L - 1]).sum())
    ev = np.array([(rr[lo:hi] * disc[:hi - lo]).sum() for lo, hi in zip(off[:-1], off[1:])])
    return j_steps, ret.sum(1), cov, np.array(subsets), float(np.mean(ev))


def magic_point(j_step_returns, cov, subset_returns):
    """The bias-variance SLSQP combination of the j-step returns."""
    n = len(subset_returns)
    m, se = np.mean(subset_returns), scipy.stats.sem(subset_returns)
    h = se * scipy.stats.t._ppf((1 + CONF) / 2.0, n - 1)
    lo, hi = m - h, m + h
    bias = np.where(j_step_returns < lo, lo - j_step_returns,
                    np.where(j_step_returns > hi, j_step_returns - hi, 0.0))
    error = cov + bias * bias
    J = len(j_step_returns)
    res = scipy.optimize.minimize(lambda x, e: x @ e @ x, np.zeros(J), args=error,
                                  constraints={"type": "eq", "fun": lambda x: np.sum(x) - 1.0},
                                  bounds=[(0, 1)] * J)
    return float(np.dot(np.array(res.x), j_step_returns))
