"""SequentialDoublyRobustEstimator (reagent/evaluation/sequential_doubly_robust_estimator.py):
one thread per episode of the sorted page runs the float32 recursion of :76-96 on rb200_ope_sdr."""
import logging

import numpy as np
import torch

from . import _ope
from .cpe import CpeEstimate, bootstrapped_std_error_of_mean

logger = logging.getLogger(__name__)


def episode_estimates(edp, gamma):
    """(per-episode doubly-robust values, per-episode discounted returns), float32 [E] each."""
    assert edp.mdp_id is not None
    ep = _ope.episodes(edp)
    prop = _ope.f32(edp.model_propensities, "model_propensities")
    n, A = prop.shape
    qv = _ope.f32(edp.model_values, "model_values")
    am = _ope.f32(edp.action_mask, "action_mask")
    r = _ope.f32(edp.logged_rewards, "logged_rewards").reshape(-1)
    lp = _ope.f32(edp.logged_propensities, "logged_propensities").reshape(-1)
    if qv.shape != (n, A) or am.shape != (n, A) or r.numel() != n or lp.numel() != n:
        raise ValueError("SequentialDoublyRobustEstimator: inconsistent page shapes")
    ep_dr = torch.empty(ep.num, device=prop.device)
    ep_val = torch.empty(ep.num, device=prop.device)
    _ope._call("rb200_ope_sdr", ep.num, ep.off.data_ptr(), A, prop.data_ptr(), qv.data_ptr(),
               am.data_ptr(), r.data_ptr(), lp.data_ptr(), float(gamma), ep_dr.data_ptr(),
               ep_val.data_ptr())
    return ep_dr, ep_val


class SequentialDoublyRobustEstimator:
    def __init__(self, gamma, rng: str = "numpy"):
        self.gamma = gamma
        self.rng = rng

    def estimate(self, edp) -> CpeEstimate:
        # For details, visit https://arxiv.org/pdf/1511.03722.pdf
        ep_dr, ep_val = episode_estimates(edp, self.gamma)
        dr_score = float(np.mean(ep_dr.cpu().numpy().astype(np.float64)))
        # the reference bootstraps a float64 array of the per-episode values
        dr_score_std_error = bootstrapped_std_error_of_mean(ep_dr.double(), rng=self.rng)
        logged_policy_score = np.mean(ep_val.cpu().numpy().astype(np.float64))
        if logged_policy_score < 1e-6:
            logger.warning("Can't normalize SDR-CPE because of small or negative "
                           f"logged_policy_score ({logged_policy_score}).")
            return CpeEstimate(raw=dr_score, normalized=0.0, raw_std_error=dr_score_std_error,
                               normalized_std_error=0.0)
        return CpeEstimate(raw=dr_score, normalized=dr_score / logged_policy_score,
                           raw_std_error=dr_score_std_error,
                           normalized_std_error=dr_score_std_error / logged_policy_score)
