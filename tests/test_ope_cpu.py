"""Counterfactual policy evaluation without a GPU: the numpy oracle against the goldens of
oracle/make_ope_golden.py, the host half of weighted DR / MAGIC, the np.random stream and the
refusals that happen before any launch."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import ope_oracle as O

GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ope_*.npz"))
                if not os.path.basename(p).startswith("ope_trainer_"))
IDS = [os.path.basename(p)[:-4] for p in GOLDEN]


def scores(d):
    """(k, logged rewards, model values, model rewards) of each scored column of the sorted page."""
    o = d["sorted_order"]
    A = d["in_action_mask"].shape[1]
    out = [(0, d["in_logged_rewards"][o], d["in_model_values"][o], d["in_model_rewards"][o])]
    if "in_logged_metrics" in d.files:
        for i in range(d["in_logged_metrics"].shape[1]):
            out.append((i + 1, d["in_logged_metrics"][o][:, i:i + 1],
                        d["in_model_metrics_values"][o][:, i * A:(i + 1) * A],
                        d["in_model_metrics"][o][:, i * A:(i + 1) * A]))
    return out


def test_goldens_present():
    assert len(GOLDEN) >= 8


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_oracle_reproduces_golden(path):
    d = np.load(path)
    o = d["sorted_order"]
    assert np.array_equal(o, O.sort_order(d["in_mdp_id"], d["in_sequence_number"]))
    g = float(d["gamma"])
    mdp, seq = d["in_mdp_id"][o], d["in_sequence_number"][o]
    assert np.array_equal(O.logged_values(d["in_logged_rewards"][o], mdp, seq, g),
                          d["sorted_logged_values"])
    if "in_logged_metrics" in d.files:
        assert np.array_equal(O.logged_values(d["in_logged_metrics"][o], mdp, seq, g),
                              d["sorted_logged_metrics_values"])
    prop, am, lp = d["in_model_propensities"][o], d["in_action_mask"][o], d["in_logged_propensities"][o]
    for k, r, qv, mr in scores(d):
        if f"sdr_{k}" not in d.files:
            continue
        drs, _ = O.sdr_episodes(prop, qv, am, r, lp, mdp, g)
        assert np.array_equal(drs.astype(np.float64), d[f"sdr_{k}"])
        if f"wsdr_{k}_returns" not in d.files:  # one episode: no confidence subsets
            with pytest.raises(ZeroDivisionError):
                O.wsdr_stats(prop, qv, am, r, lp, mdp, g, 25)
            continue
        _, jr, cov, sub, _ = O.wsdr_stats(prop, qv, am, r, lp, mdp, g, 25)
        np.testing.assert_allclose(jr, d[f"wsdr_{k}_returns"], rtol=1e-5, atol=1e-12)
        np.testing.assert_allclose(cov, d[f"wsdr_{k}_cov"], rtol=1e-5,
                                   atol=1e-7 * np.abs(d[f"wsdr_{k}_cov"]).max())
        np.testing.assert_allclose(sub, d[f"wsdr_{k}_subsets"], rtol=2e-5)
        if f"est_{k}" in d.files:
            # set_metric_as_reward keeps the reward's model_rewards_for_logged_action
            dm, ips, dr = O.dr_rows(prop, mr, am, r, d["in_model_rewards_for_logged_action"][o], lp)
            raw = d[f"est_{k}"][:, 0]
            np.testing.assert_allclose([dm.mean(), ips.mean(), dr.mean()], raw[:3], rtol=1e-5)
            np.testing.assert_allclose(drs.astype(np.float64).mean(), raw[3], rtol=1e-6)
            np.testing.assert_allclose(jr[0], raw[4], rtol=1e-5)


@pytest.mark.parametrize("path", [p for p in GOLDEN if "est_0" in np.load(p).files],
                         ids=[i for p, i in zip(GOLDEN, IDS) if "est_0" in np.load(p).files])
def test_host_magic_combination_matches_golden(path):
    """The SLSQP combination of the golden's j-step statistics gives the golden MAGIC point
    estimate exactly (the host half of the estimator, fed the reference's inputs)."""
    from reagent_b200.evaluation.weighted_sequential_doubly_robust_estimator import \
        WeightedSequentialDoublyRobustEstimator as W

    d = np.load(path)
    for k in range(3):
        if f"est_{k}" not in d.files:
            break
        jr, cov, sub = d[f"wsdr_{k}_returns"], d[f"wsdr_{k}_cov"], list(d[f"wsdr_{k}_subsets"])
        got = W.blend(jr, cov, sub)
        assert got == d[f"est_{k}"][5][0]
        assert O.magic_point(jr, cov, np.array(sub)) == got


def test_numpy_choice_draws_randint():
    """np.random.choice(data, n, replace=True) consumes the stream as randint(0, len, n): the
    bootstrap's host indices leave np.random where the reference leaves it."""
    data = np.arange(37, dtype=np.float32)
    np.random.seed(5)
    a = np.random.choice(data, 11, replace=True)
    s1 = np.random.get_state()
    np.random.seed(5)
    b = data[np.random.randint(0, len(data), 11)]
    s2 = np.random.get_state()
    assert np.array_equal(a, b) and np.array_equal(s1[1], s2[1]) and s1[2] == s2[2]


def test_refuses_host_tensors_and_bad_ids():
    from reagent_b200 import _lib
    from reagent_b200.evaluation import _ope

    with pytest.raises(_lib.Rb200Error):
        _ope.f32(torch.zeros(3, 2), "x")
    with pytest.raises(_lib.Rb200Error):
        _ope.check_ids(torch.zeros(3, 1, dtype=torch.int64), torch.zeros(3, 1, dtype=torch.int64))


def test_refuses_non_dqn_input():
    from reagent_b200.core import types as rlt
    from reagent_b200.evaluation import EvaluationDataPage

    with pytest.raises(NotImplementedError):
        EvaluationDataPage.create_from_training_batch(object(), None)
    assert hasattr(rlt, "DiscreteDqnInput")


def test_evaluator_rejects_unknown_rng():
    from reagent_b200.evaluation import Evaluator

    with pytest.raises(ValueError):
        Evaluator(["a", "b"], 0.9, None, rng="python")
