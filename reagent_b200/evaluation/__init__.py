"""Counterfactual policy evaluation of discrete-action policies (reagent/evaluation/): the
EvaluationDataPage of a validation set and the Evaluator's DM, IPS, DR, sequential DR, weighted DR
and MAGIC estimates, computed on the device by the kernels of csrc/rb200_ope.cu; and the world-model
LossEvaluator, FeatureImportanceEvaluator and FeatureSensitivityEvaluator on csrc/rb200_mdnrnn.cu."""
from .cpe import CpeDetails, CpeEstimate, CpeEstimateSet, bootstrapped_std_error_of_mean
from .doubly_robust_estimator import DoublyRobustEstimator, DoublyRobustHP
from .evaluation_data_page import EvaluationDataPage
from .evaluator import Evaluator
from .sequential_doubly_robust_estimator import SequentialDoublyRobustEstimator
from .weighted_sequential_doubly_robust_estimator import WeightedSequentialDoublyRobustEstimator
from .world_model_evaluator import (FeatureImportanceEvaluator, FeatureSensitivityEvaluator,
                                    LossEvaluator)

__all__ = ["CpeDetails", "CpeEstimate", "CpeEstimateSet", "bootstrapped_std_error_of_mean",
           "DoublyRobustEstimator", "DoublyRobustHP", "EvaluationDataPage", "Evaluator",
           "SequentialDoublyRobustEstimator", "WeightedSequentialDoublyRobustEstimator",
           "LossEvaluator", "FeatureImportanceEvaluator", "FeatureSensitivityEvaluator"]
