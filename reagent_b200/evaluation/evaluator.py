"""Evaluator (reagent/evaluation/evaluator.py:56-143): every CPE estimate of a sorted page with
logged values, for the reward and for each metric in metrics_to_score.  `rng` selects the index
stream of the bootstrapped standard errors: "numpy" draws them from the global np.random stream
as the reference does (so the stream afterwards is the reference's), "device" draws them in the
kernel from torch's CUDA generator (reproducible under torch.manual_seed)."""
import logging
from .cpe import CpeDetails, CpeEstimateSet
from .doubly_robust_estimator import DoublyRobustEstimator
from .sequential_doubly_robust_estimator import SequentialDoublyRobustEstimator
from .weighted_sequential_doubly_robust_estimator import WeightedSequentialDoublyRobustEstimator

logger = logging.getLogger(__name__)


class Evaluator:
    NUM_J_STEPS_FOR_MAGIC_ESTIMATOR = 25

    def __init__(self, action_names, gamma, model, metrics_to_score=None, rng: str = "numpy"):
        if rng not in ("numpy", "device"):
            raise ValueError(f"rng must be 'numpy' or 'device', got {rng!r}")
        self.action_names = action_names
        self.metrics_to_score = metrics_to_score
        self.gamma = gamma
        self.model = model
        self.rng = rng
        self.doubly_robust_estimator = DoublyRobustEstimator(rng=rng)
        self.sequential_doubly_robust_estimator = SequentialDoublyRobustEstimator(gamma, rng=rng)
        self.weighted_sequential_doubly_robust_estimator = WeightedSequentialDoublyRobustEstimator(gamma)

    def evaluate_post_training(self, edp) -> CpeDetails:
        cpe_details = CpeDetails()
        cpe_details.reward_estimates = self.score_cpe("Reward", edp)
        if (self.metrics_to_score is not None and edp.logged_metrics is not None
                and self.action_names is not None):
            for i, metric in enumerate(self.metrics_to_score):
                logger.info("--------- Running CPE on metric: {} ---------".format(metric))
                metric_reward_edp = edp.set_metric_as_reward(i, len(self.action_names))
                cpe_details.metric_estimates[metric] = self.score_cpe(metric, metric_reward_edp)
        if self.action_names is not None:
            if edp.optimal_q_values is not None:
                value_means = edp.optimal_q_values.mean(dim=0).tolist()
                cpe_details.q_value_means = {
                    action: float(value_means[i]) for i, action in enumerate(self.action_names)}
                value_stds = edp.optimal_q_values.std(dim=0).tolist()
                cpe_details.q_value_stds = {
                    action: float(value_stds[i]) for i, action in enumerate(self.action_names)}
            if edp.eval_action_idxs is not None:
                counts = [int(c) for c in (edp.eval_action_idxs.reshape(-1, 1) == edp.eval_action_idxs.new_tensor(
                    range(len(self.action_names)))).sum(dim=0).tolist()]
                n = edp.eval_action_idxs.shape[0]
                cpe_details.action_distribution = {
                    action: float(counts[i]) / n for i, action in enumerate(self.action_names)}
        return cpe_details

    def score_cpe(self, metric_name, edp) -> CpeEstimateSet:
        direct_method, inverse_propensity, doubly_robust = self.doubly_robust_estimator.estimate(edp)
        sequential_doubly_robust = self.sequential_doubly_robust_estimator.estimate(edp)
        weighted_doubly_robust = self.weighted_sequential_doubly_robust_estimator.estimate(
            edp, num_j_steps=1, whether_self_normalize_importance_weights=True)
        magic = self.weighted_sequential_doubly_robust_estimator.estimate(
            edp, num_j_steps=Evaluator.NUM_J_STEPS_FOR_MAGIC_ESTIMATOR,
            whether_self_normalize_importance_weights=True)
        return CpeEstimateSet(
            direct_method=direct_method, inverse_propensity=inverse_propensity,
            doubly_robust=doubly_robust, sequential_doubly_robust=sequential_doubly_robust,
            weighted_doubly_robust=weighted_doubly_robust, magic=magic)
