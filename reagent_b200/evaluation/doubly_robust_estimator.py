"""DoublyRobustEstimator (reagent/evaluation/doubly_robust_estimator.py:101-348): the direct
method, IPS and doubly-robust rows on rb200_ope_dr_rows, their means as fixed-order device sums,
and the three bootstrapped standard errors.  BOP-E / _split_data are not provided."""
import logging
from typing import Dict, NamedTuple, Optional, Tuple, Union

import torch

from . import _ope
from .cpe import CpeEstimate, bootstrapped_std_error_of_mean

logger = logging.getLogger(__name__)

DEFAULT_FRAC_TRAIN = 0.4
DEFAULT_FRAC_VALID = 0.1


class DoublyRobustHP(NamedTuple):
    frac_train: float = DEFAULT_FRAC_TRAIN
    frac_valid: float = DEFAULT_FRAC_VALID
    bootstrap_num_samples: int = 1000
    bootstrap_sample_percent: float = 0.25
    xgb_params: Optional[Dict[str, Union[float, int, str]]] = None
    bope_mode: Optional[str] = None
    bope_num_samples: Optional[int] = None


def _estimate(score, std_error, normalizer):
    return CpeEstimate(raw=score, normalized=score * normalizer, raw_std_error=std_error,
                       normalized_std_error=std_error * normalizer)


class DoublyRobustEstimator:
    """For details, visit https://arxiv.org/pdf/1612.01205.pdf"""

    def __init__(self, rng: str = "numpy"):
        self.rng = rng

    def estimate(self, edp, hp: Optional[DoublyRobustHP] = None
                 ) -> Tuple[CpeEstimate, CpeEstimate, CpeEstimate]:
        hp = hp or DoublyRobustHP()
        prop = _ope.f32(edp.model_propensities, "model_propensities")
        n, A = prop.shape
        mr = _ope.f32(edp.model_rewards, "model_rewards")
        am = _ope.f32(edp.action_mask, "action_mask")
        r = _ope.f32(edp.logged_rewards, "logged_rewards")
        mrl = _ope.f32(edp.model_rewards_for_logged_action, "model_rewards_for_logged_action")
        lp = _ope.f32(edp.logged_propensities, "logged_propensities")
        if mr.shape != (n, A) or am.shape != (n, A) or not (r.shape == mrl.shape == lp.shape == (n, 1)):
            raise ValueError("DoublyRobustEstimator: inconsistent page shapes")
        dm, ips, dr = (torch.empty(n, device=prop.device) for _ in range(3))
        _ope._call("rb200_ope_dr_rows", n, A, prop.data_ptr(), mr.data_ptr(), am.data_ptr(),
                   r.data_ptr(), mrl.data_ptr(), lp.data_ptr(), dm.data_ptr(), ips.data_ptr(),
                   dr.data_ptr())
        # mean logged reward: normalises every estimate (0 when it is too small to divide by)
        logged_policy_score = _ope.mean(r)
        if logged_policy_score < 1e-6:
            logger.warning("Can't normalize DR-CPE because of small or negative logged_policy_score")
            normalizer = 0.0
        else:
            normalizer = 1.0 / logged_policy_score

        def std(x):
            return bootstrapped_std_error_of_mean(x, sample_percent=hp.bootstrap_sample_percent,
                                                  num_samples=hp.bootstrap_num_samples, rng=self.rng)

        dm_std = std(dm)
        direct_method = _estimate(_ope.mean(dm), dm_std, normalizer)
        ips_std = std(ips)
        inverse_propensity = _estimate(_ope.mean(ips), ips_std, normalizer)
        dr_std = std(dr)
        doubly_robust = _estimate(_ope.mean(dr), dr_std, normalizer)
        return direct_method, inverse_propensity, doubly_robust
