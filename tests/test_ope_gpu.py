"""Counterfactual policy evaluation on the GPU against the goldens of oracle/make_ope_golden.py
(the unmodified reference's sort, compute_values, validate and Evaluator) and the numpy oracle."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import ope_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ope_*.npz"))
                if not os.path.basename(p).startswith("ope_trainer_"))
IDS = [os.path.basename(p)[:-4] for p in GOLDEN]
EST = ("direct_method", "inverse_propensity", "doubly_robust", "sequential_doubly_robust",
       "weighted_doubly_robust", "magic")


def page_from(d, dev="cuda"):
    from reagent_b200.evaluation import EvaluationDataPage

    f = {k[3:]: torch.from_numpy(d[k]).to(dev) for k in d.files if k.startswith("in_")}
    A = f["action_mask"].shape[1]
    if "model_metrics" not in f:
        f["model_metrics"] = torch.zeros(f["model_rewards"].shape[0], 0, device=dev)
    return EvaluationDataPage(**f), A


def prepared(d):
    edp, A = page_from(d)
    edp = edp.sort().compute_values(float(d["gamma"]))
    edp.validate()
    return edp, A


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_sorted_page_and_logged_values_bit_exact(path):
    d = np.load(path)
    edp, _ = prepared(d)
    o = d["sorted_order"]
    assert np.array_equal(edp.mdp_id.cpu().numpy(), d["in_mdp_id"][o])
    assert np.array_equal(edp.model_propensities.cpu().numpy(), d["in_model_propensities"][o])
    assert np.array_equal(edp.logged_values.cpu().numpy(), d["sorted_logged_values"])
    if "sorted_logged_metrics_values" in d.files:
        assert np.array_equal(edp.logged_metrics_values.cpu().numpy(),
                              d["sorted_logged_metrics_values"])


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_sdr_episodes_bit_exact_and_wsdr_statistics(path):
    from reagent_b200.evaluation.sequential_doubly_robust_estimator import episode_estimates
    from reagent_b200.evaluation.weighted_sequential_doubly_robust_estimator import j_step_statistics

    d = np.load(path)
    edp, A = prepared(d)
    pages = [edp] + [edp.set_metric_as_reward(i, A)
                     for i in range(0 if edp.logged_metrics is None else edp.logged_metrics.shape[1])]
    for k, p in enumerate(pages):
        ep_dr, _ = episode_estimates(p, float(d["gamma"]))
        assert np.array_equal(ep_dr.cpu().numpy().astype(np.float64), d[f"sdr_{k}"])
        if f"wsdr_{k}_returns" not in d.files:  # one episode: no confidence subsets
            with pytest.raises(ZeroDivisionError):
                j_step_statistics(p, float(d["gamma"]), 25)
            continue
        _, jr, cov, sub, _, _ = j_step_statistics(p, float(d["gamma"]), 25)
        np.testing.assert_allclose(jr, d[f"wsdr_{k}_returns"], rtol=1e-5, atol=1e-12)
        np.testing.assert_allclose(cov, d[f"wsdr_{k}_cov"], rtol=1e-5,
                                   atol=1e-7 * np.abs(d[f"wsdr_{k}_cov"]).max())
        np.testing.assert_allclose(sub, d[f"wsdr_{k}_subsets"], rtol=2e-5)


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_evaluate_post_training_matches_reference(path):
    from reagent_b200.evaluation import Evaluator

    d = np.load(path)
    edp, A = prepared(d)
    K = 0 if edp.logged_metrics is None else edp.logged_metrics.shape[1]
    ev = Evaluator([str(a) for a in range(A)], float(d["gamma"]), None,
                   metrics_to_score=[f"m{i}" for i in range(K)] or None)
    np.random.seed(int(d["np_seed"]))
    if str(d["error"]):
        with pytest.raises(Exception) as e:
            ev.evaluate_post_training(edp)
        assert type(e.value).__name__ == str(d["error"])
    else:
        details = ev.evaluate_post_training(edp)
    state = np.random.get_state()
    assert np.array_equal(state[1], d["rng_keys"]) and state[2] == int(d["rng_pos"])
    if str(d["error"]):
        return
    sets = [details.reward_estimates] + [details.metric_estimates[f"m{i}"] for i in range(K)]
    for k, s in enumerate(sets):
        want = d[f"est_{k}"]
        for row, name in enumerate(EST):
            tol = 1e-4 if name == "magic" else 1e-5
            np.testing.assert_allclose(np.array(getattr(s, name), dtype=np.float64), want[row],
                                       rtol=tol, atol=1e-9, err_msg=f"{name} of score {k}")


def test_repeat_is_deterministic():
    from reagent_b200.evaluation import Evaluator

    d = np.load(GOLDEN[IDS.index("ope_mixed")])
    edp, A = prepared(d)
    ev = Evaluator([str(a) for a in range(A)], 0.9, None)
    outs = []
    for _ in range(2):
        np.random.seed(3)
        outs.append(ev.score_cpe("Reward", edp))
    assert outs[0] == outs[1]


def test_malformed_episodes_raise():
    d = np.load(GOLDEN[IDS.index("ope_mixed")])
    edp, _ = prepared(d)
    seq = edp.sequence_number.clone()
    seq[1] = seq[0]
    with pytest.raises(AssertionError, match="increasing"):
        edp._replace(sequence_number=seq).validate()
    mdp = edp.mdp_id.clone()
    mdp[-1] = mdp[0]
    with pytest.raises(AssertionError, match="broken up"):
        edp._replace(mdp_id=mdp).validate()
    with pytest.raises(ValueError):
        edp._replace(mdp_id=edp.mdp_id.int()).compute_values(0.9)


def synthetic_page(n, A=8, seed=0, dev="cuda"):
    from reagent_b200.evaluation import EvaluationDataPage

    g = torch.Generator(device=dev).manual_seed(seed)
    lens = torch.randint(1, 31, (n // 15 + 1,), generator=g, device=dev)
    lens = lens[: int((torch.cumsum(lens, 0) < n).sum()) + 1]
    n = int(lens.sum())
    mdp = torch.repeat_interleave(torch.arange(lens.numel(), device=dev), lens).reshape(-1, 1)
    seq = (torch.arange(n, device=dev) - torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens)).reshape(-1, 1)
    act = torch.randint(0, A, (n,), generator=g, device=dev)
    am = torch.nn.functional.one_hot(act, A).float()
    prop = torch.softmax(torch.randn(n, A, generator=g, device=dev), 1)
    r = torch.randn(n, 1, generator=g, device=dev) + 0.5
    mr = torch.randn(n, A, generator=g, device=dev) + 0.5
    return EvaluationDataPage(
        mdp_id=mdp, sequence_number=seq, logged_propensities=torch.rand(n, 1, generator=g, device=dev) * 0.8 + 0.1,
        logged_rewards=r, action_mask=am, model_propensities=prop, model_rewards=mr,
        model_rewards_for_logged_action=(mr * am).sum(1, keepdim=True),
        model_values=torch.randn(n, A, generator=g, device=dev) + 0.5,
        model_metrics=torch.zeros(n, 0, device=dev))


def test_million_rows_against_oracle():
    from reagent_b200.evaluation.doubly_robust_estimator import DoublyRobustEstimator
    from reagent_b200.evaluation.sequential_doubly_robust_estimator import episode_estimates
    from reagent_b200.evaluation.weighted_sequential_doubly_robust_estimator import (
        WeightedSequentialDoublyRobustEstimator as W, j_step_statistics)

    edp = synthetic_page(1_000_000).sort().compute_values(0.9)
    h = {k: getattr(edp, k).cpu().numpy() for k in ("mdp_id", "model_propensities", "model_values",
                                                     "action_mask", "logged_rewards",
                                                     "logged_propensities", "model_rewards",
                                                     "model_rewards_for_logged_action")}
    dm, ips, dr = O.dr_rows(h["model_propensities"], h["model_rewards"], h["action_mask"],
                            h["logged_rewards"], h["model_rewards_for_logged_action"],
                            h["logged_propensities"])
    est = DoublyRobustEstimator().estimate(edp)
    np.testing.assert_allclose([e.raw for e in est], [dm.astype(np.float64).mean(),
                                                      ips.astype(np.float64).mean(),
                                                      dr.astype(np.float64).mean()], rtol=1e-5)
    ep_dr, _ = episode_estimates(edp, 0.9)
    drs, _ = O.sdr_episodes(h["model_propensities"], h["model_values"], h["action_mask"],
                            h["logged_rewards"], h["logged_propensities"], h["mdp_id"], 0.9)
    assert np.array_equal(ep_dr.cpu().numpy(), drs)
    _, jr, cov, sub, _, _ = j_step_statistics(edp, 0.9, 25)
    _, ojr, ocov, osub, _ = O.wsdr_stats(h["model_propensities"], h["model_values"],
                                         h["action_mask"], h["logged_rewards"],
                                         h["logged_propensities"], h["mdp_id"], 0.9, 25)
    np.testing.assert_allclose(jr, ojr, rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(cov, ocov, rtol=1e-5, atol=1e-7 * np.abs(ocov).max())
    np.testing.assert_allclose(sub, osub, rtol=1e-5, atol=1e-12)
    # weighted DR is the infinite-step return; MAGIC's point estimate blends all 25
    np.testing.assert_allclose(jr[0], ojr[0], rtol=1e-5)
    np.testing.assert_allclose(W.blend(jr, cov, sub), O.magic_point(ojr, ocov, osub), rtol=1e-4)


def test_device_rng_reproducible_and_calibrated():
    from reagent_b200.evaluation import bootstrapped_std_error_of_mean

    sigma, n = 2.0, 200_000
    data = torch.randn(n, device="cuda") * sigma
    torch.manual_seed(11)
    a = bootstrapped_std_error_of_mean(data, rng="device")
    torch.manual_seed(11)
    b = bootstrapped_std_error_of_mean(data, rng="device")
    c = bootstrapped_std_error_of_mean(data, rng="device")
    assert a == b and a != c
    expect = float(data.std()) / np.sqrt(int(0.25 * n))
    assert abs(a / expect - 1) < 0.10, (a, expect)


def _dqn_trainer(S=6, A=4, K=1):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import DQNTrainer

    torch.manual_seed(0)
    q = FullyConnectedDQN(S, A, [16], ["relu"])
    rn = FullyConnectedDQN(S, (K + 1) * A, [16], ["relu"])
    qc = FullyConnectedDQN(S, (K + 1) * A, [16], ["relu"])
    return DQNTrainer(q.cuda(), q.get_target_network().cuda(), rn.cuda(), qc.cuda(),
                      qc.get_target_network().cuda(), metrics_to_score=[f"m{i}" for i in range(K)],
                      actions=[str(a) for a in range(A)], rl=RLParameters(gamma=0.9),
                      evaluation=EvaluationParameters(calc_cpe_in_training=True)).cuda()


def _batch(n, S=6, A=4, K=1, seed=0):
    from reagent_b200.core import types as rlt

    g = torch.Generator().manual_seed(seed)
    act = torch.nn.functional.one_hot(torch.randint(0, A, (n,), generator=g), A).float()
    mdp = torch.randint(0, n // 5 + 1, (n, 1), generator=g)
    seq = (torch.arange(n) + seed * n).reshape(-1, 1)  # pages of one epoch continue the episodes
    return rlt.DiscreteDqnInput(
        state=rlt.FeatureData(torch.randn(n, S, generator=g)),
        next_state=rlt.FeatureData(torch.randn(n, S, generator=g)),
        action=act, next_action=act.roll(1, 0), reward=torch.randn(n, 1, generator=g) + 1,
        time_diff=torch.ones(n, 1), step=None, not_terminal=torch.ones(n, 1), possible_actions_mask=torch.ones(n, A),
        possible_next_actions_mask=torch.ones(n, A),
        extras=rlt.ExtraData(mdp_id=mdp, sequence_number=seq,
                             action_probability=torch.rand(n, 1, generator=g) * 0.5 + 0.25,
                             metrics=torch.randn(n, K, generator=g))).cuda()


def test_dqn_validation_step_and_epoch_end():
    from reagent_b200.evaluation import CpeDetails, EvaluationDataPage

    t = _dqn_trainer()
    logged = []

    class Reporter:
        def log(self, **kw):
            logged.append(kw)

    t.set_reporter(Reporter())
    pages = [t.validation_step(_batch(300, seed=s), s) for s in range(2)]
    assert all(isinstance(p, EvaluationDataPage) and p.model_propensities.is_cuda for p in pages)
    x = _batch(300, seed=0).state.float_features
    q, _ = t.get_detached_model_outputs(x)
    assert torch.equal(pages[0].optimal_q_values, q)
    np.random.seed(0)
    t.validation_epoch_end(pages)
    details = [kw["cpe_details"] for kw in logged if "cpe_details" in kw]
    assert len(details) == 1 and isinstance(details[0], CpeDetails)
    d = details[0]
    d.reward_estimates.check_estimates_exist()
    d.metric_estimates["m0"].check_estimates_exist()
    assert abs(sum(d.action_distribution.values()) - 1) < 1e-9


TRAINER_GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ope_trainer_*.npz")))
TRAINER_IDS = [os.path.basename(p)[12:-4] for p in TRAINER_GOLDEN]
PAGE_FIELDS = ("logged_propensities", "logged_rewards", "action_mask", "model_propensities",
               "model_rewards", "model_rewards_for_logged_action", "model_values",
               "possible_actions_mask", "optimal_q_values", "eval_action_idxs", "logged_metrics",
               "model_metrics", "model_metrics_for_logged_action", "model_metrics_values",
               "model_metrics_values_for_logged_action")


def _page_kernel(q, r_out, c_out, mask, action, reward, boosts, temperature):
    from reagent_b200.evaluation import _ope

    n, A = q.shape
    K = r_out.shape[1] // A - 1
    out = dict(boosted=torch.empty(n, 1, device="cuda"), prop=torch.empty(n, A, device="cuda"),
               idx=torch.empty(n, 1, dtype=torch.int64, device="cuda"),
               mr=torch.empty(n, 1, device="cuda"), mm=torch.empty(n, K, device="cuda"),
               mmv=torch.empty(n, K, device="cuda"))
    _ope._call("rb200_ope_page", n, A, K, q.data_ptr(), r_out.data_ptr(), c_out.data_ptr(),
               mask.data_ptr(), action.data_ptr(), reward.data_ptr(), boosts.data_ptr(),
               float(temperature), out["boosted"].data_ptr(), out["prop"].data_ptr(),
               out["idx"].data_ptr(), out["mr"].data_ptr(), out["mm"].data_ptr(), out["mmv"].data_ptr())
    return out


def _cpe_heads_propensities(q, mask, action, temperature, M):
    """propensities_next of rb200_cpe_heads with next_scores = q and the same mask."""
    from reagent_b200 import _lib

    n, A = q.shape
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    keep = dict(mr=z(n, M), nt=torch.ones(n, device="cuda"), re=z(n, M * A), qc=z(n, M * A),
                qt=z(n, M * A), dr=z(n, M * A), dq=z(n, M * A), p=z(n, A),
                lp=z(2 * ((n + 255) // 256)), loss=z(2),
                cnt=torch.zeros(1, dtype=torch.int32, device="cuda"))
    a = _lib.CpeArgsT()
    a.batch, a.num_actions, a.num_metrics = n, A, M
    a.next_scores, a.mask, a.temperature = q.data_ptr(), mask.data_ptr(), float(temperature)
    a.action, a.metrics_reward, a.gamma = action.data_ptr(), keep["mr"].data_ptr(), 0.9
    a.discount_src, a.discount_mode = None, _lib.DISCOUNT_CONST
    a.not_terminal, a.reward_est = keep["nt"].data_ptr(), keep["re"].data_ptr()
    a.qcpe, a.qcpe_target_next = keep["qc"].data_ptr(), keep["qt"].data_ptr()
    a.loss_kind = _lib.LOSS_MSE
    a.dz_reward, a.dz_qcpe = keep["dr"].data_ptr(), keep["dq"].data_ptr()
    a.propensities_next, a.loss_partials = keep["p"].data_ptr(), keep["lp"].data_ptr()
    a.loss, a.tile_counter = keep["loss"].data_ptr(), keep["cnt"].data_ptr()
    _lib.check(_lib.lib().rb200_cpe_heads(a, _lib.cur_stream()), "rb200_cpe_heads")
    return keep["p"]


@pytest.mark.parametrize("path", TRAINER_GOLDEN, ids=TRAINER_IDS)
def test_page_kernel_on_reference_network_outputs(path):
    """rb200_ope_page fed the reference's own network outputs: boosted rewards, eval_action_idxs
    and every logged-action gather bit for bit; propensities bit for bit against rb200_cpe_heads
    and within float32 rounding of torch's CPU masked_softmax."""
    d = np.load(path)
    t = lambda k: torch.from_numpy(np.ascontiguousarray(d[k])).float().cuda()  # noqa: E731
    q, mask, action = t("out_q"), t("batch_possible_actions_mask"), t("batch_action")
    out = _page_kernel(q, t("out_r"), t("out_c"), mask, action, t("batch_reward"), t("boosts"),
                       float(d["temperature"]))
    assert np.array_equal(out["boosted"].cpu().numpy(), d["page_logged_rewards"])
    assert np.array_equal(out["idx"].cpu().numpy(), d["page_eval_action_idxs"])
    assert np.array_equal(out["mr"].cpu().numpy(), d["page_model_rewards_for_logged_action"])
    assert np.array_equal(out["mm"].cpu().numpy(), d["page_model_metrics_for_logged_action"])
    assert np.array_equal(out["mmv"].cpu().numpy(), d["page_model_metrics_values_for_logged_action"])
    M = d["out_r"].shape[1] // q.shape[1]
    assert torch.equal(out["prop"], _cpe_heads_propensities(q, mask, action, float(d["temperature"]), M))
    np.testing.assert_allclose(out["prop"].cpu().numpy(), d["page_model_propensities"],
                               rtol=1e-6, atol=1e-7)


def _trainer_from(d, kind):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import (DuelingQNetwork, FullyConnectedActor, FullyConnectedDQN,
                                     FullyConnectedNetwork)
    from reagent_b200.training import DiscreteCRRTrainer, DQNTrainer
    from reagent_b200.training.dqn_trainer import BCQConfig

    S, A = d["batch_state"].shape[1], d["batch_action"].shape[1]
    M = d["out_r"].shape[1] // A

    def load(m, name):
        sd = {k[len(name) + 4:]: torch.from_numpy(d[k]) for k in d.files
              if k.startswith(f"sd.{name}.")}
        m.load_state_dict(sd)
        return m.cuda()

    boosts = d["boosts"]
    rl = RLParameters(gamma=float(d["gamma"]), temperature=float(d["temperature"]),
                      reward_boost={str(a): float(b) for a, b in enumerate(boosts) if b} or None)
    rn = load(FullyConnectedDQN(S, M * A, [16], ["relu"]), "r")
    qc = load(FullyConnectedDQN(S, M * A, [16], ["relu"]), "c")
    common = dict(metrics_to_score=[f"m{i}" for i in range(M - 1)],
                  actions=[str(a) for a in range(A)], rl=rl,
                  evaluation=EvaluationParameters(calc_cpe_in_training=True))
    if kind == "crr":
        actor = load(FullyConnectedActor(S, A, [16], ["relu"]), "actor")
        q1 = load(FullyConnectedDQN(S, A, [16], ["relu"]), "q1")
        return DiscreteCRRTrainer(
            actor_network=actor, actor_network_target=actor.get_target_network(), q1_network=q1,
            q1_network_target=q1.get_target_network(), reward_network=rn, q_network_cpe=qc,
            q_network_cpe_target=qc.get_target_network(), **common).cuda()
    q = (DuelingQNetwork.make_fully_connected(S, A, [16], ["relu"]) if kind == "dueling"
         else FullyConnectedDQN(S, A, [16], ["relu"]))
    q = load(q, "q")
    extra = {}
    if kind == "bcq":
        extra = dict(imitator=load(FullyConnectedNetwork([S, 8, A], ["relu", "linear"]), "im"),
                     bcq=BCQConfig(drop_threshold=0.1))
    return DQNTrainer(q, q.get_target_network(), rn, qc, qc.get_target_network(), **common,
                      **extra).cuda()


def _golden_rlt_batch(d):
    from reagent_b200.core import types as rlt

    b = {k[6:]: torch.from_numpy(d[k]).cuda() for k in d.files if k.startswith("batch_")}
    n = b["state"].shape[0]
    return rlt.DiscreteDqnInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["state"]),
        reward=b["reward"], time_diff=torch.ones(n, 1, device="cuda"), step=None,
        not_terminal=torch.ones(n, 1, device="cuda"), action=b["action"], next_action=b["action"],
        possible_actions_mask=b["possible_actions_mask"],
        possible_next_actions_mask=b["possible_actions_mask"],
        extras=rlt.ExtraData(mdp_id=b["mdp_id"], sequence_number=b["sequence_number"],
                             action_probability=b["action_probability"], metrics=b["metrics"]))


@pytest.mark.parametrize("path", TRAINER_GOLDEN, ids=TRAINER_IDS)
def test_trainer_page_and_cpe_details_match_reference(path):
    """The page of a trainer loaded with the reference's weights (DQNTrainer.validation_step, or
    create_from_training_batch for CRR), then validation_epoch_end's CpeDetails."""
    from reagent_b200.evaluation import EvaluationDataPage

    d = np.load(path)
    kind = os.path.basename(path)[12:-4]
    t = _trainer_from(d, kind)
    batch = _golden_rlt_batch(d)
    page = (EvaluationDataPage.create_from_training_batch(batch, t) if kind == "crr"
            else t.validation_step(batch, 0))
    assert page.model_propensities.is_cuda
    for f in PAGE_FIELDS:
        got, want = getattr(page, f), d["page_" + f]
        got = got.cpu().numpy()
        assert got.shape == want.shape, f
        if f == "eval_action_idxs" or f in ("logged_propensities", "logged_rewards", "action_mask",
                                            "possible_actions_mask", "logged_metrics"):
            assert np.array_equal(got, want), f
        else:
            np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * np.abs(want).max(), err_msg=f)
    logged = []

    class Reporter:
        def log(self, **kw):
            logged.append(kw)

    t.set_reporter(Reporter())
    np.random.seed(int(d["np_seed"]))
    t.validation_epoch_end([page])
    state = np.random.get_state()
    assert np.array_equal(state[1], d["rng_keys"]) and state[2] == int(d["rng_pos"])
    [details] = [kw["cpe_details"] for kw in logged if "cpe_details" in kw]
    A = d["batch_action"].shape[1]
    sets = [details.reward_estimates] + [details.metric_estimates[f"m{i}"]
                                         for i in range(d["out_r"].shape[1] // A - 1)]
    for k, s in enumerate(sets):
        # The page's network outputs are the GPU forward's, a few float32 ulps from the
        # reference's CPU forward; weighted DR multiplies up to 20 importance ratios and sums
        # terms of both signs, so its error is bounded against the scale of the score's
        # estimates, not against its own (possibly small) value.
        scale = np.abs(d[f"est_{k}"][:, 0]).max()
        for row, name in enumerate(EST):
            tol = 1e-4 if name == "magic" else 1e-5
            np.testing.assert_allclose(np.array(getattr(s, name), dtype=np.float64),
                                       d[f"est_{k}"][row], rtol=tol, atol=1e-5 * scale,
                                       err_msg=f"{name} of score {k}")
    acts = [str(a) for a in range(A)]
    np.testing.assert_allclose([details.q_value_means[a] for a in acts], d["cpe_q_means"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose([details.q_value_stds[a] for a in acts], d["cpe_q_stds"], rtol=1e-5, atol=1e-6)
    assert [details.action_distribution[a] for a in acts] == list(d["cpe_action_dist"])
