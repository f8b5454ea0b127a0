"""Write tests/golden/ope_*.npz from the UNMODIFIED reference evaluation code (reagent/evaluation/),
imported through oracle/ref_harness.py.  Each case builds an EvaluationDataPage from seeded
tensors, then runs the reference's sort, compute_values, validate and
Evaluator.evaluate_post_training with a seeded np.random stream.  Recorded per case:
  in_*        the unsorted page fields
  sorted_*    the sorted page with its logged values (and the sort order)
  sdr_<k>     the per-episode sequential-DR values of score k (0 = reward, i = metric i)
  wsdr_<k>_*  MAGIC's j-step returns, covariance and subset infinite-step returns of score k
  est_<k>     every CpeEstimate of score k, rows DM, IPS, DR, SDR, WDR, MAGIC
  rng_*       the np.random state after the call
The trainer cases (ope_trainer_*) build the page with the reference's
EvaluationDataPage.create_from_training_batch from a seeded trainer with CPE heads (plain,
dueling, BCQ, reward boost, discrete CRR) and also record
  sd.<net>.<key>  the state dict of each network the page reads
  batch_*         the batch; out_q / out_r / out_c the reference's network outputs
  page_*          every page field; cpe_q_means / cpe_q_stds / cpe_action_dist
Usage: python oracle/make_ope_golden.py  (rewrites the files byte for byte)."""
import io
import os
import sys
import zipfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_harness import ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
FIELDS = ("mdp_id", "sequence_number", "logged_propensities", "logged_rewards", "action_mask",
          "model_propensities", "model_rewards", "model_rewards_for_logged_action", "model_values",
          "logged_metrics", "model_metrics", "model_metrics_values")
EST = ("direct_method", "inverse_propensity", "doubly_robust", "sequential_doubly_robust",
       "weighted_doubly_robust", "magic")


def make_page(seed, lengths, A=4, K=0, reward_shift=0.5, zero_prop_step=None, shuffle=True):
    """A page of len(lengths) episodes; rows shuffled; K metrics."""
    g = torch.Generator().manual_seed(seed)
    n = int(sum(lengths))
    mdp = torch.cat([torch.full((L,), 1000 + 7 * e, dtype=torch.int64) for e, L in enumerate(lengths)])
    seq = torch.cat([torch.cumsum(torch.randint(1, 3, (L,), generator=g), 0) for L in lengths])
    act = torch.randint(0, A, (n,), generator=g)
    action_mask = torch.nn.functional.one_hot(act, A).float()
    logits = torch.randn(n, A, generator=g)
    model_propensities = torch.softmax(logits, dim=1)
    if zero_prop_step is not None:  # the model never takes the logged action at that step
        first = torch.cat([torch.tensor([0]), torch.cumsum(torch.tensor(lengths), 0)[:-1]])
        rows = first[torch.tensor(lengths) > zero_prop_step] + zero_prop_step
        model_propensities[rows] = model_propensities[rows] * (1 - action_mask[rows])
    logged_propensities = torch.rand(n, 1, generator=g) * 0.8 + 0.1
    M = K + 1
    rewards_all = torch.randn(n, M, generator=g) + reward_shift
    model_all = torch.randn(n, M * A, generator=g) + reward_shift
    values_all = torch.randn(n, M * A, generator=g) * 2 + reward_shift
    page = dict(
        mdp_id=mdp.reshape(-1, 1), sequence_number=seq.reshape(-1, 1),
        logged_propensities=logged_propensities, logged_rewards=rewards_all[:, :1].contiguous(),
        action_mask=action_mask, model_propensities=model_propensities,
        model_rewards=model_all[:, :A].contiguous(),
        model_rewards_for_logged_action=(model_all[:, :A] * action_mask).sum(1, keepdim=True),
        model_values=values_all[:, :A].contiguous())
    if K:
        page["logged_metrics"] = rewards_all[:, 1:].contiguous()
        page["model_metrics"] = model_all[:, A:].contiguous()
        page["model_metrics_values"] = values_all[:, A:].contiguous()
    if shuffle:
        perm = torch.randperm(n, generator=g)
        page = {k: v[perm] for k, v in page.items()}
    return page


CASES = {
    "ope_mixed": dict(seed=1, lengths=None, A=8),
    "ope_len1": dict(seed=2, lengths=[1] * 300, A=4),
    "ope_long": dict(seed=3, lengths=[3, 1, 200, 2, 5, 4, 1, 2, 3, 6], A=3),
    "ope_metrics2": dict(seed=4, lengths=None, A=5, K=2),
    "ope_where_zeros": dict(seed=5, lengths=[4, 6, 5, 7, 3, 8, 6, 5], A=4, zero_prop_step=2),
    "ope_negative": dict(seed=6, lengths=None, A=4, reward_shift=-1.0),
    "ope_two": dict(seed=7, lengths=[5, 3], A=4),
    "ope_three": dict(seed=8, lengths=[4, 2, 6], A=4),
    "ope_one": dict(seed=9, lengths=[7], A=4),
}

TRAINER_CASES = {
    "ope_trainer_dqn": dict(kind="dqn", seed=11, A=4),
    "ope_trainer_dueling": dict(kind="dueling", seed=12, A=8),
    "ope_trainer_bcq": dict(kind="bcq", seed=13, A=5),
    "ope_trainer_boost": dict(kind="boost", seed=14, A=5, temperature=0.5),
    "ope_trainer_crr": dict(kind="crr", seed=15, A=4),
}
PAGE_FIELDS = ("logged_propensities", "logged_rewards", "action_mask", "model_propensities",
               "model_rewards", "model_rewards_for_logged_action", "model_values",
               "possible_actions_mask", "optimal_q_values", "eval_action_idxs", "logged_metrics",
               "model_metrics", "model_metrics_for_logged_action", "model_metrics_values",
               "model_metrics_values_for_logged_action")


def trainer_case(name, *, kind, seed, A, S=7, n=240, K=1, sizes=(16,), acts=("relu",),
                 temperature=0.1):
    """A reference trainer with CPE heads, a batch of ~24 shuffled episodes, its page and the
    Evaluator's CpeDetails after gather_eval_data."""
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    dqn_mod = ref("reagent.models.dqn")
    evaluator_mod = ref("reagent.evaluation.evaluator")
    EDP = ref("reagent.evaluation.evaluation_data_page").EvaluationDataPage
    torch.manual_seed(seed)
    sizes, acts = list(sizes), list(acts)
    n_out = (K + 1) * A

    def perturbed(m):
        with torch.no_grad():
            for p in m.parameters():
                if p.dim() == 1:
                    p.normal_(0, 0.1)
        return m

    reward_net = perturbed(dqn_mod.FullyConnectedDQN(S, n_out, sizes, acts))
    qcpe = perturbed(dqn_mod.FullyConnectedDQN(S, n_out, sizes, acts))
    metrics = [f"m{i}" for i in range(K)]
    boost = {"0": 0.25, str(A - 1): -0.5} if kind == "boost" else None
    rl = params.RLParameters(gamma=0.9, temperature=temperature, reward_boost=boost)
    ev_params = params.EvaluationParameters(calc_cpe_in_training=True)
    actions = [str(a) for a in range(A)]
    nets = {"r": reward_net, "c": qcpe}
    if kind == "crr":
        actor_mod = ref("reagent.models.actor")
        tr = ref("reagent.training.discrete_crr_trainer")
        actor = perturbed(actor_mod.FullyConnectedActor(S, A, sizes, acts))
        q1 = perturbed(dqn_mod.FullyConnectedDQN(S, A, sizes, acts))
        trainer = tr.DiscreteCRRTrainer(
            actor_network=actor, actor_network_target=actor.get_target_network(), q1_network=q1,
            q1_network_target=q1.get_target_network(), reward_network=reward_net,
            q_network_cpe=qcpe, q_network_cpe_target=qcpe.get_target_network(),
            metrics_to_score=metrics, evaluation=ev_params, rl=rl, actions=actions)
        nets.update(actor=actor, q1=q1)
    else:
        tr = ref("reagent.training.dqn_trainer")
        if kind == "dueling":
            duel = ref("reagent.models.dueling_q_network")
            q = perturbed(duel.DuelingQNetwork.make_fully_connected(S, A, sizes, acts))
        else:
            q = perturbed(dqn_mod.FullyConnectedDQN(S, A, sizes, acts))
        extra = {}
        if kind == "bcq":
            fcn = ref("reagent.models.fully_connected_network")
            im = perturbed(fcn.FullyConnectedNetwork([S, 8, A], ["relu", "linear"]))
            extra = dict(imitator=im, bcq=tr.BCQConfig(drop_threshold=0.1))
            nets["im"] = im
        trainer = tr.DQNTrainer(q, q.get_target_network(), reward_net, qcpe,
                                qcpe.get_target_network(), metrics_to_score=metrics,
                                actions=actions, rl=rl, evaluation=ev_params, **extra)
        nets["q"] = q
    g = torch.Generator().manual_seed(seed + 1)
    lengths = torch.randint(1, 21, (n,), generator=g)
    lengths = lengths[: int((torch.cumsum(lengths, 0) < n).sum())]
    lengths = torch.cat((lengths, torch.tensor([n - int(lengths.sum())])))
    lengths = lengths[lengths > 0]
    mdp = torch.repeat_interleave(torch.arange(len(lengths)) * 3 + 5, lengths)
    seq = torch.cat([torch.cumsum(torch.randint(1, 3, (int(L),), generator=g), 0) for L in lengths])
    pam = (torch.rand(n, A, generator=g) > 0.3).float()
    act_idx = torch.randint(A, (n,), generator=g)
    pam[torch.arange(n), act_idx] = 1.0
    perm = torch.randperm(n, generator=g)
    batch = dict(state=torch.randn(n, S, generator=g), action=torch.nn.functional.one_hot(act_idx, A).float(),
                 reward=torch.randn(n, 1, generator=g) + 0.5, possible_actions_mask=pam,
                 mdp_id=mdp.reshape(-1, 1), sequence_number=seq.reshape(-1, 1),
                 action_probability=torch.rand(n, 1, generator=g) * 0.7 + 0.2,
                 metrics=torch.randn(n, K, generator=g) + 0.5)
    batch = {k: v[perm] for k, v in batch.items()}
    rb = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(batch["state"]), next_state=rlt.FeatureData(batch["state"]),
        reward=batch["reward"], time_diff=torch.ones(n, 1), step=None,
        not_terminal=torch.ones(n, 1), action=batch["action"], next_action=batch["action"],
        possible_actions_mask=batch["possible_actions_mask"],
        possible_next_actions_mask=batch["possible_actions_mask"],
        extras=rlt.ExtraData(mdp_id=batch["mdp_id"], sequence_number=batch["sequence_number"],
                             action_probability=batch["action_probability"],
                             metrics=batch["metrics"]))
    arrays = {"batch_" + k: v.numpy() for k, v in batch.items()}
    for net_name, m in nets.items():
        for k, v in m.state_dict().items():
            arrays[f"sd.{net_name}.{k}"] = v.numpy()
    with torch.no_grad():
        x = rlt.FeatureData(batch["state"])
        arrays["out_q"] = trainer.get_detached_model_outputs(x)[0].numpy()
        arrays["out_r"] = reward_net(x).numpy()
        arrays["out_c"] = qcpe(x).numpy()
    page = EDP.create_from_training_batch(rb, trainer)
    for f in PAGE_FIELDS:
        v = getattr(page, f)
        if v is not None:
            arrays["page_" + f] = v.numpy()
    arrays["boosts"] = trainer.reward_boosts.numpy().reshape(-1)
    arrays["temperature"] = np.array(float(trainer.rl_temperature))
    arrays["gamma"] = np.array(0.9)
    arrays["np_seed"] = np.array(seed + 100)
    eval_data = trainer.gather_eval_data([page])
    np.random.seed(seed + 100)
    details = trainer.evaluator.evaluate_post_training(eval_data)
    state = np.random.get_state()
    arrays["rng_keys"] = state[1]
    arrays["rng_pos"] = np.array(state[2])
    sets = [details.reward_estimates] + [details.metric_estimates[m] for m in metrics]
    for k, est_set in enumerate(sets):
        arrays[f"est_{k}"] = np.array([[float(v) for v in getattr(est_set, e)] for e in EST])
    arrays["cpe_q_means"] = np.array([details.q_value_means[a] for a in actions])
    arrays["cpe_q_stds"] = np.array([details.q_value_stds[a] for a in actions])
    arrays["cpe_action_dist"] = np.array([details.action_distribution[a] for a in actions])
    return arrays


def run_case(name, spec):
    EDP = ref("reagent.evaluation.evaluation_data_page").EvaluationDataPage
    evaluator_mod = ref("reagent.evaluation.evaluator")
    sdr_mod = ref("reagent.evaluation.sequential_doubly_robust_estimator")
    wsdr_mod = ref("reagent.evaluation.weighted_sequential_doubly_robust_estimator")
    spec = dict(spec)
    seed = spec["seed"]
    if spec["lengths"] is None:
        rs = np.random.RandomState(seed)
        spec["lengths"] = [int(x) for x in rs.randint(1, 31, 40)]
    K = spec.get("K", 0)
    page = make_page(**spec)
    arrays = {"in_" + k: v.numpy() for k, v in page.items()}
    gamma = 0.9
    edp = EDP(**page, model_metrics_values_for_logged_action=None,
              model_metrics_for_logged_action=None, logged_values=None, logged_metrics_values=None)
    if not K:
        edp = edp._replace(model_metrics=torch.zeros(edp.model_rewards.shape[0], 0))
    edp = edp.sort()
    edp = edp.compute_values(gamma)
    edp.validate()
    order = sorted(range(len(page["mdp_id"])),
                   key=lambda i: (int(page["mdp_id"][i]), int(page["sequence_number"][i]), i))
    arrays["sorted_order"] = np.array(order, dtype=np.int64)
    arrays["sorted_logged_values"] = edp.logged_values.numpy()
    if K:
        arrays["sorted_logged_metrics_values"] = edp.logged_metrics_values.numpy()
    # record the per-episode SDR values and MAGIC's j-step statistics as the reference computes them
    rec = {"sdr": [], "wsdr": []}
    orig_boot = sdr_mod.bootstrapped_std_error_of_mean

    def boot(data, *a, **k):
        rec["sdr"].append(np.array(data, dtype=np.float64))
        return orig_boot(data, *a, **k)

    orig_point = wsdr_mod.WeightedSequentialDoublyRobustEstimator.compute_weighted_doubly_robust_point_estimate

    def point(self, j_steps, num_j_steps, j_step_returns, infinite_step_returns,
              j_step_return_trajectories):
        if len(rec["wsdr"]) < len(rec["sdr"]):
            rec["wsdr"].append((np.array(j_step_returns), np.cov(j_step_return_trajectories),
                                np.array(infinite_step_returns)))
        return orig_point(self, j_steps, num_j_steps, j_step_returns, infinite_step_returns,
                          j_step_return_trajectories)

    sdr_mod.bootstrapped_std_error_of_mean = boot
    wsdr_mod.WeightedSequentialDoublyRobustEstimator.compute_weighted_doubly_robust_point_estimate = point
    metrics = [f"m{i}" for i in range(K)] or None
    ev = evaluator_mod.Evaluator([str(a) for a in range(spec.get("A", 4))], gamma, None,
                                 metrics_to_score=metrics)
    np.random.seed(seed + 100)
    try:
        details = ev.evaluate_post_training(edp)
        arrays["error"] = np.array("")
    except (ZeroDivisionError, ValueError) as e:  # the reference fails on 1 and 2 episodes
        details = None
        arrays["error"] = np.array(type(e).__name__)
    finally:
        sdr_mod.bootstrapped_std_error_of_mean = orig_boot
        wsdr_mod.WeightedSequentialDoublyRobustEstimator.compute_weighted_doubly_robust_point_estimate = orig_point
    state = np.random.get_state()
    arrays["rng_keys"] = state[1]
    arrays["rng_pos"] = np.array(state[2])
    arrays["gamma"] = np.array(gamma)
    arrays["np_seed"] = np.array(seed + 100)
    for k, d in enumerate(rec["sdr"]):
        arrays[f"sdr_{k}"] = d
    for k, (jr, cov, inf) in enumerate(rec["wsdr"]):
        arrays[f"wsdr_{k}_returns"] = jr
        arrays[f"wsdr_{k}_cov"] = cov
        arrays[f"wsdr_{k}_subsets"] = inf
    if details is not None:
        sets = [details.reward_estimates] + [details.metric_estimates[m] for m in metrics or []]
        for k, s in enumerate(sets):
            arrays[f"est_{k}"] = np.array([[float(v) for v in getattr(s, e)] for e in EST])
    return arrays


def write_npz(path, arrays):
    """np.savez with fixed zip timestamps, so the bytes depend on the arrays only."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    torch.set_num_threads(1)
    for name, spec in CASES.items():
        write_npz(os.path.join(OUT, name + ".npz"), run_case(name, spec))
        print("wrote", name)
    for name, spec in TRAINER_CASES.items():
        write_npz(os.path.join(OUT, name + ".npz"), trainer_case(name, **spec))
        print("wrote", name)


if __name__ == "__main__":
    main()
