"""WeightedSequentialDoublyRobustEstimator (reagent/evaluation/
weighted_sequential_doubly_robust_estimator.py): weighted DR and MAGIC.

The reference pads every episode to the longest one; here the page stays in episode (CSR)
layout.  rb200_ope_wsdr_rows takes the cumulative importance weights, rb200_ope_seg_sum their
per-time-step sums (over all trajectories, and within each of the confidence subsets), and
rb200_ope_wsdr_returns every j-step return of every trajectory in one walk, from which the
j-step sums, np.cov and the subsets' infinite-step returns follow.  Only the SLSQP combination
over at most 25 weights, the confidence bounds and MAGIC's 50 subset draws run on the host."""
import logging

import numpy as np
import scipy as sp
import scipy.optimize  # noqa: F401
import scipy.stats  # noqa: F401
import torch

from .. import _lib
from . import _ope
from .cpe import CpeEstimate

logger = logging.getLogger(__name__)


def _row_statistics(edp):
    """Per-row cumulative importance weights, V(s) and Q(s, a_log) of the page, the time step
    and trajectory of every row, and the weights' per-time-step sums.  Computed once per page
    object: weighted DR and MAGIC of one score share them."""
    cache = edp.__dict__.setdefault("_wsdr_rows", {})
    if cache:
        return cache
    ep = _ope.episodes(edp)
    prop = _ope.f32(edp.model_propensities, "model_propensities")
    n, A = prop.shape
    qv = _ope.f32(edp.model_values, "model_values")
    am = _ope.f32(edp.action_mask, "action_mask")
    lp = _ope.f32(edp.logged_propensities, "logged_propensities").reshape(-1)
    if qv.shape != (n, A) or am.shape != (n, A) or lp.numel() != n:
        raise ValueError("WeightedSequentialDoublyRobustEstimator: inconsistent page shapes")
    dev = prop.device
    lens = ep.lengths()
    L = int(lens.max())
    # shorter episodes are padded in the reference, which turns its arrays into float64
    fp64 = int(int(lens.min()) != L)
    T = torch.float64 if fp64 else torch.float32
    w, sv, ql = (torch.empty(n, dtype=T, device=dev) for _ in range(3))
    _ope._call("rb200_ope_wsdr_rows", ep.num, ep.off.data_ptr(), A, fp64, prop.data_ptr(),
               qv.data_ptr(), am.data_ptr(), lp.data_ptr(), w.data_ptr(), sv.data_ptr(),
               ql.data_ptr())
    traj = torch.repeat_interleave(torch.arange(ep.num, device=dev), lens)
    step = torch.arange(n, device=dev) - ep.off[:-1].long()[traj]
    cache.update(ep=ep, L=L, fp64=fp64, T=T, w=w, sv=sv, ql=ql, traj=traj, step=step,
                 r=_ope.f32(edp.logged_rewards, "logged_rewards").reshape(-1))
    cache["col"] = _col_sums(cache, step, L)
    return cache


def _col_sums(rows, key, nseg):
    """Sums of the raw weights over the rows of each key value, in a fixed order."""
    dev = key.device
    perm = torch.argsort(key, stable=True)
    seg_off = torch.zeros(nseg + 1, dtype=torch.int64, device=dev)
    seg_off[1:] = torch.cumsum(torch.bincount(key, minlength=nseg), 0)
    return _ope.seg_sum(rows["w"], seg_off, perm)


def j_step_statistics(edp, gamma, num_j_steps):
    """(j_steps, the j-step returns summed over trajectories [J], their covariance over
    trajectories [J, J] (None for one j-step), the confidence subsets' infinite-step returns,
    the mean discounted logged return, the number of trajectories) of the page."""
    rows = _row_statistics(edp)
    ep, L, dev, T = rows["ep"], rows["L"], rows["w"].device, rows["T"]
    E = ep.num
    j_steps = [float("inf")] + ([-1] if num_j_steps > 1 else [])
    if num_j_steps > 2:
        stride = L // (num_j_steps - 1)
        j_steps += [stride * i for i in range(1, num_j_steps - 1)]
    J = len(j_steps)
    if J > _lib.OPE_MAX_J:
        raise ValueError(f"num_j_steps is limited to {_lib.OPE_MAX_J}")
    bounds = [0]
    if J > 1:
        S = int(min(E / 2, WeightedSequentialDoublyRobustEstimator.NUM_SUBSETS_FOR_CB_ESTIMATES))
        width = E / S  # a single trajectory has no subsets: ZeroDivisionError, as in the reference
        bounds = [int(width * i) for i in range(S + 1)]
    S = len(bounds) - 1
    sub_off = torch.tensor(bounds, dtype=torch.int32, device=dev)
    if S:
        sub = torch.searchsorted(sub_off[1:].long(), rows["traj"], right=True)
        key = torch.where(sub < S, sub * L + rows["step"], torch.full_like(rows["step"], S * L))
        sub_col = _col_sums(rows, key, S * L + 1)
    else:
        sub_col = torch.zeros(1, dtype=T, device=dev)
    js = torch.tensor([int(min(j, L - 1)) for j in j_steps], dtype=torch.int32, device=dev)
    disc = torch.from_numpy(np.logspace(0, L - 1, L, base=gamma)).to(dev)
    ret = torch.empty(J, E, dtype=torch.float64, device=dev)
    sub_ret = torch.empty(E, dtype=torch.float64, device=dev)
    ev = torch.empty(E, dtype=torch.float64, device=dev)
    _ope._call("rb200_ope_wsdr_returns", E, ep.off.data_ptr(), rows["fp64"], rows["w"].data_ptr(),
               rows["sv"].data_ptr(), rows["ql"].data_ptr(), rows["r"].data_ptr(),
               disc.data_ptr(), L, rows["col"].data_ptr(), J, js.data_ptr(), S,
               sub_off.data_ptr(), sub_col.data_ptr(), ret.data_ptr(), sub_ret.data_ptr(),
               ev.data_ptr())
    totals = _ope.seg_sum(ret.reshape(-1), torch.arange(J + 1, device=dev) * E).cpu().numpy()
    cov = None
    if J > 1:
        cov = torch.empty(J, J, dtype=torch.float64, device=dev)
        _ope._call("rb200_ope_cov", ret.data_ptr(), J, E, cov.data_ptr())
        cov = cov.cpu().numpy()
    subset_returns = _ope.seg_sum(sub_ret, sub_off.long()).cpu().numpy() if S else np.zeros(0)
    score = float(_ope.seg_sum(ev, torch.tensor([0, E], device=dev)).item()) / E
    return j_steps, totals, cov, list(subset_returns), score, E


class WeightedSequentialDoublyRobustEstimator:
    """Weighted sequential DR (num_j_steps=1) and MAGIC (Thomas & Brunskill 2016, sections 5, 7
    and 8) with self-normalised importance weights."""

    NUM_SUBSETS_FOR_CB_ESTIMATES = 25
    CONFIDENCE_INTERVAL = 0.9
    NUM_BOOTSTRAP_SAMPLES = 50
    BOOTSTRAP_SAMPLE_PCT = 0.5

    def __init__(self, gamma):
        self.gamma = gamma

    def estimate(self, edp, num_j_steps, whether_self_normalize_importance_weights) -> CpeEstimate:
        if edp.model_values is None:
            raise ValueError("weighted DR needs model_values")
        if not whether_self_normalize_importance_weights:
            raise NotImplementedError("only self-normalised importance weights are supported")
        _, returns, cov, subset_returns, score, _ = j_step_statistics(edp, self.gamma, num_j_steps)
        if len(returns) == 1:
            value, spread = returns[0], 0.0
        else:
            value = self.blend(returns, cov, subset_returns)
            # the spread of the blend over random halves of the subsets' worth of j-steps
            k = int(self.BOOTSTRAP_SAMPLE_PCT * len(subset_returns))
            blends = []
            for _ in range(self.NUM_BOOTSTRAP_SAMPLES):
                pick = np.sort(np.random.choice(num_j_steps, k, replace=False))
                blends.append(self.blend(returns[pick], cov[np.ix_(pick, pick)], subset_returns))
            spread = np.std(blends)
        if score < 1e-6:
            logger.warning("Can't normalize WSDR-CPE because of small or negative logged_policy_score")
            return CpeEstimate(raw=value, normalized=0.0, raw_std_error=spread,
                               normalized_std_error=0.0)
        return CpeEstimate(raw=value, normalized=value / score, raw_std_error=spread,
                           normalized_std_error=spread / score)

    @classmethod
    def blend(cls, returns, cov, subset_returns):
        """MAGIC's combination: the weights x >= 0, sum 1, minimising x' (cov + b^2) x, where b is
        how far each j-step return lies outside the subsets' confidence interval (broadcast
        over rows, as the reference adds it); returns x . returns."""
        lo, hi = cls.confidence_bounds(subset_returns, cls.CONFIDENCE_INTERVAL)
        b = np.maximum(lo - returns, 0.0) + np.maximum(returns - hi, 0.0)
        err = cov + b * b
        J = len(returns)
        sol = sp.optimize.minimize(lambda x, e: x @ e @ x, np.zeros(J), args=err,
                                   constraints={"type": "eq", "fun": lambda x: x.sum() - 1.0},
                                   bounds=[(0, 1)] * J)
        return float(np.asarray(sol.x) @ returns)

    @staticmethod
    def confidence_bounds(x, confidence):
        """Student-t interval of the mean of x at the two-sided level `confidence`."""
        half = sp.stats.sem(x) * sp.stats.t._ppf(0.5 + confidence / 2.0, len(x) - 1)
        return np.mean(x) - half, np.mean(x) + half
