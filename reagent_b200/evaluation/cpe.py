"""CpeEstimate, CpeEstimateSet, CpeDetails and bootstrapped_std_error_of_mean
(reagent/evaluation/cpe.py)."""
import logging
from typing import Dict, NamedTuple, Optional

import numpy as np
import torch

from . import _ope

logger = logging.getLogger(__name__)


class CpeEstimate(NamedTuple):
    raw: float
    normalized: float
    raw_std_error: float
    normalized_std_error: float


class CpeEstimateSet(NamedTuple):
    direct_method: Optional[CpeEstimate] = None
    inverse_propensity: Optional[CpeEstimate] = None
    doubly_robust: Optional[CpeEstimate] = None

    sequential_doubly_robust: Optional[CpeEstimate] = None
    weighted_doubly_robust: Optional[CpeEstimate] = None
    magic: Optional[CpeEstimate] = None

    switch: Optional[CpeEstimate] = None
    switch_dr: Optional[CpeEstimate] = None

    def check_estimates_exist(self):
        for name in ("direct_method", "inverse_propensity", "doubly_robust",
                     "sequential_doubly_robust", "weighted_doubly_robust", "magic"):
            assert getattr(self, name) is not None, name

    def log(self):
        self.check_estimates_exist()
        for label, e in (("Reward Inverse Propensity Score", self.inverse_propensity),
                         ("Reward Direct Method", self.direct_method),
                         ("Reward Doubly Robust P.E.", self.doubly_robust),
                         ("Value Weighted Doubly Robust P.E.", self.weighted_doubly_robust),
                         ("Value Sequential Doubly Robust P.E.", self.sequential_doubly_robust),
                         ("Value Magic Doubly Robust P.E.", self.magic)):
            logger.info(f"{label} : normalized {e.normalized:.3f} +/- {e.normalized_std_error:.3f} "
                        f"raw {e.raw:.3f} +/- {e.raw_std_error:.3f}")

    def fill_empty_with_zero(self):
        """This set with every missing estimate replaced by an all-zero CpeEstimate."""
        zero = CpeEstimate(0.0, 0.0, 0.0, 0.0)
        return CpeEstimateSet(*(zero if e is None else e for e in self))


class CpeDetails:
    def __init__(self):
        self.reward_estimates: CpeEstimateSet = CpeEstimateSet()
        self.metric_estimates: Dict[str, CpeEstimateSet] = {}
        self.q_value_means: Optional[Dict[str, float]] = None
        self.q_value_stds: Optional[Dict[str, float]] = None
        self.action_distribution: Optional[Dict[str, float]] = None

    def log(self):
        logger.info("Reward Estimates:")
        logger.info("-----------------")
        self.reward_estimates.log()
        logger.info("-----------------")
        for metric in self.metric_estimates.keys():
            logger.info(metric + " Estimates:")
            logger.info("-----------------")
            self.metric_estimates[metric].log()
            logger.info("-----------------")


def bootstrapped_std_error_of_mean(data, sample_percent=0.25, num_samples=1000, rng="numpy"):
    """Bootstrapped standard error of the mean of `data` (a 1-D tensor or array; host data is
    copied to the current CUDA device): the std of `num_samples` means of samples of
    int(sample_percent * len(data)) elements drawn with replacement.  The means are computed on
    the device in float64 and, for float32 data, rounded to float32 as numpy's mean of a float32
    sample is; the std is then taken in that precision.  See _ope.bootstrap_means for the two
    index streams."""
    fp64 = (data.dtype == torch.float64 if isinstance(data, torch.Tensor)
            else np.asarray(data).dtype == np.float64)
    if not isinstance(data, torch.Tensor) or data.device.type != "cuda":
        data = torch.as_tensor(np.asarray(data)).cuda()
    sample_size = int(sample_percent * len(data))
    means = _ope.bootstrap_means(data, sample_size, num_samples, rng)
    return np.std(means if fp64 else means.astype(np.float32))
