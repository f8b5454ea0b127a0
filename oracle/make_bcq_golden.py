"""Generate the batch-constrained Q-learning (BCQ) golden vectors in tests/golden/ by running the
UNMODIFIED reference (DQNTrainer with an imitator and BCQConfig, BatchConstrainedDQN) through
oracle/ref_harness.py.  Needs the reference checkout (build container only); the files are
committed.

    python oracle/make_bcq_golden.py            # regenerate every BCQ case
    python oracle/make_bcq_golden.py NAME ...   # only the named ones

The DQN cases draw exactly what oracle/make_golden.py's dqn_case draws, in the same order, and
then the imitator; each holds the usual DQN arrays plus
  im.W*/im.b*                 imitator weights (a bare FullyConnectedNetwork: `.dnn`, no `.fc`)
  bcq.r_state, bcq.r_next_state   the reference's filter values r = softmax / its row max
  bcq.next_mask0              the filtered next-action mask of update 0
  after.possible_*_mask       the batch masks after the run (the reference's `*=` writes them)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import N_UPDATES, _dump_net, _fc_params, _np, _perturb, _save  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402


def _dump_dnn(arrays, prefix, module):
    """A bare FullyConnectedNetwork (no `.fc` wrapper), e.g. a BCQ imitator."""
    for i, seq in enumerate(module.dnn):
        arrays[f"{prefix}.W{i}"] = _np(seq[0].weight).copy()
        arrays[f"{prefix}.b{i}"] = _np(seq[0].bias).copy()


def _make_imitator(S, A, sizes, scale):
    """BCQ imitator as the reference's tests build it (reagent/test/models/test_bcq.py):
    FullyConnectedNetwork([S, ..., A], [..., "linear"]), biases perturbed, last layer scaled so
    that a sizeable share of the actions falls below the drop threshold."""
    fcn = ref("reagent.models.fully_connected_network")
    im = fcn.FullyConnectedNetwork([S] + list(sizes) + [A], ["relu"] * len(sizes) + ["linear"])
    with torch.no_grad():
        for seq in im.dnn:
            seq[0].bias.normal_(0, 0.1)
        im.dnn[-1][0].weight.mul_(scale)
        im.dnn[-1][0].bias.mul_(scale)
    return im


def _filter_values(im, x):
    """r of get_valid_actions_from_imitator (reagent/training/imitator_training.py:17-24)."""
    with torch.no_grad():
        p = torch.nn.functional.softmax(im(x), dim=1)
        return p / p.max(keepdim=True, dim=1)[0]


def _check_margin(r, thr, what):
    """No filter value within fp32 noise of the threshold (it would flip on rounding alone, which
    is not a parity question), and 30-70 % of the actions dropped."""
    rel = ((r - thr).abs() / thr).min().item()
    drop = (r < thr).float().mean().item()
    assert rel > 1e-4, f"{what}: a filter value lies {rel:.2e} (relative) from the threshold"
    assert 0.3 <= drop <= 0.7, f"{what}: {drop:.0%} of the actions dropped"


def bcq_dqn_case(name, *, bcq, B=48, S=12, A=5, sizes=(24, 20), acts=("relu", "relu"),
                 loss="huber", double_q=True, multi_steps=None, boost=None, random_masks=False,
                 gamma=0.97, tau=0.05, lr=1e-2, seed=0, dueling=False, cpe_metrics=None,
                 temperature=0.01, imitator_sizes=(16,), imitator_scale=4.0):
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    dqn_mod = ref("reagent.models.dqn")
    tr = ref("reagent.training.dqn_trainer")
    union = ref("reagent.optimizer.union")
    torch.manual_seed(seed)
    if dueling:
        duel = ref("reagent.models.dueling_q_network")
        q = duel.DuelingQNetwork.make_fully_connected(S, A, list(sizes), list(acts))
    else:
        q = dqn_mod.FullyConnectedDQN(S, A, list(sizes), list(acts))
    with torch.no_grad():
        for _, b in _fc_params(q):
            b.normal_(0, 0.1)
    qt = q.get_target_network()
    with torch.no_grad():
        for w, b in _fc_params(qt):
            w.add_(torch.randn_like(w) * 0.05)
            b.add_(torch.randn_like(b) * 0.05)
    A_names = [str(i) for i in range(A)]
    rl = params.RLParameters(gamma=gamma, target_update_rate=tau, q_network_loss=loss,
                             maxq_learning=True, multi_steps=multi_steps,
                             reward_boost=boost, temperature=temperature)
    cpe = cpe_metrics is not None
    reward_net = qcpe = qcpe_t = None
    if cpe:
        n_out = (len(cpe_metrics) + 1) * A
        reward_net = dqn_mod.FullyConnectedDQN(S, n_out, list(sizes), list(acts))
        qcpe = dqn_mod.FullyConnectedDQN(S, n_out, list(sizes), list(acts))
        with torch.no_grad():
            for net in (reward_net, qcpe):
                for _, b in _fc_params(net):
                    b.normal_(0, 0.1)
        qcpe_t = qcpe.get_target_network()
        with torch.no_grad():
            for w, b in _fc_params(qcpe_t):
                w.add_(torch.randn_like(w) * 0.05)
                b.add_(torch.randn_like(b) * 0.05)
    act_idx = torch.randint(A, (B,))
    nact_idx = torch.randint(A, (B,))
    not_terminal = (torch.rand(B, 1) > 0.2).float()
    pnam = torch.ones(B, A)
    if random_masks:
        pnam = (torch.rand(B, A) > 0.3).float()
        pnam[torch.arange(B), torch.randint(A, (B,))] = 1.0
    batch = dict(
        state=torch.randn(B, S), next_state=torch.randn(B, S), reward=torch.randn(B, 1),
        time_diff=torch.randint(1, 4, (B, 1)).float(), step=torch.randint(1, 4, (B, 1)),
        not_terminal=not_terminal,
        action=torch.nn.functional.one_hot(act_idx, A).float(),
        next_action=torch.nn.functional.one_hot(nact_idx, A).float() * not_terminal,
        possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=pnam)
    if cpe:
        batch["metrics"] = torch.randn(B, len(cpe_metrics))
    # the imitator comes after every draw of the plain DQN case
    imitator = _make_imitator(S, A, imitator_sizes, imitator_scale)
    r_state = _filter_values(imitator, batch["state"])
    r_next = _filter_values(imitator, batch["next_state"])
    _check_margin(r_state, bcq, name + " state")
    _check_margin(r_next, bcq, name + " next_state")
    # the behaviour policy's favourite next action stays possible: no empty non-terminal row
    pnam[torch.arange(B), r_next.argmax(dim=1)] = 1.0
    trainer = tr.DQNTrainer(
        q, qt, reward_net, qcpe, qcpe_t, metrics_to_score=list(cpe_metrics) if cpe else None,
        actions=A_names, rl=rl, double_q_learning=double_q, minibatch_size=B,
        optimizer=union.Optimizer__Union(Adam=union.classes["Adam"](lr=lr)),
        evaluation=params.EvaluationParameters(calc_cpe_in_training=cpe),
        imitator=imitator, bcq=tr.BCQConfig(drop_threshold=bcq))
    rbatch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(batch["state"]), next_state=rlt.FeatureData(batch["next_state"]),
        reward=batch["reward"], time_diff=batch["time_diff"],
        step=batch["step"] if multi_steps is not None else None,
        not_terminal=batch["not_terminal"], action=batch["action"],
        next_action=batch["next_action"], possible_actions_mask=batch["possible_actions_mask"],
        possible_next_actions_mask=batch["possible_next_actions_mask"],
        extras=rlt.ExtraData(action_probability=torch.ones(B, 1),
                             metrics=batch.get("metrics")))
    # _np() shares memory with the tensor; the reference's in-place `mask *= keep`
    # (dqn_trainer.py:216, :291) would otherwise store the filtered masks as the inputs
    arrays = {f"batch.{k}": _np(v).copy() for k, v in batch.items()}
    _dump_net(arrays, "q0", q)
    _dump_net(arrays, "qt0", qt)
    _dump_dnn(arrays, "im", imitator)
    arrays["bcq.r_state"] = _np(r_state)
    arrays["bcq.r_next_state"] = _np(r_next)
    if cpe:
        _dump_net(arrays, "r0", reward_net)
        _dump_net(arrays, "c0", qcpe)
        _dump_net(arrays, "ct0", qcpe_t)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    assert len(opts) == (4 if cpe else 2)
    losses, cpe_losses = [], []
    for it in range(N_UPDATES):
        cap = {}
        out = run_update(trainer, rbatch, it, opts, capture=cap)
        losses.append(out[0])
        if cpe:
            cpe_losses.append([out[1], out[2]])
        if it == 0:
            for i, g in enumerate(cap[0]):
                arrays[f"grad0.{i}"] = _np(g)
            arrays["all_q0"] = _np(trainer.all_action_scores)
            # the float32 batch mask was filtered in place by update 0
            arrays["bcq.next_mask0"] = _np(batch["possible_next_actions_mask"]).copy()
            if cpe:
                for i, g in enumerate(cap[1]):
                    arrays[f"grad0r.{i}"] = _np(g)
                for i, g in enumerate(cap[2]):
                    arrays[f"grad0c.{i}"] = _np(g)
    arrays["losses"] = np.array(losses, dtype=np.float64)
    _dump_net(arrays, "qN", q)
    _dump_net(arrays, "qtN", qt)
    if cpe:
        arrays["cpe_losses"] = np.array(cpe_losses, dtype=np.float64)
        _dump_net(arrays, "rN", reward_net)
        _dump_net(arrays, "cN", qcpe)
        _dump_net(arrays, "ctN", qcpe_t)
    arrays["after.possible_next_actions_mask"] = _np(batch["possible_next_actions_mask"]).copy()
    arrays["after.possible_actions_mask"] = _np(batch["possible_actions_mask"]).copy()
    meta = dict(kind="dqn", B=B, S=S, A=A, sizes=list(sizes), acts=list(acts), loss=loss,
                double_q=double_q, maxq=True, multi_steps=multi_steps, time_diff=False,
                boost=boost, gamma=gamma, tau=tau, lr=lr, n_updates=N_UPDATES, dueling=dueling,
                cpe_metrics=cpe_metrics, temperature=temperature, bcq=bcq,
                imitator_sizes=list(imitator_sizes),
                imitator_acts=["relu"] * len(imitator_sizes) + ["linear"])
    _save(name, arrays, meta)


def bcq_model_case(name, *, B=40, S=8, A=6, sizes=(16, 12), imitator_sizes=(16,), thr=0.3,
                   imitator_scale=4.0, seed=0):
    """BatchConstrainedDQN.forward (reagent/models/bcq.py:26-35) on a batch of states."""
    rlt = ref("reagent.core.types")
    dqn_mod = ref("reagent.models.dqn")
    bcq_mod = ref("reagent.models.bcq")
    torch.manual_seed(seed)
    q = dqn_mod.FullyConnectedDQN(S, A, list(sizes), ["relu"] * len(sizes))
    _perturb(q)
    imitator = _make_imitator(S, A, imitator_sizes, imitator_scale)
    model = bcq_mod.BatchConstrainedDQN(S, q, imitator, thr)
    state = torch.randn(B, S)
    r = _filter_values(imitator, state)
    _check_margin(r, thr, name)
    with torch.no_grad():
        out = model(rlt.FeatureData(state))
        q_values = q(rlt.FeatureData(state))
    arrays = dict(state=_np(state), out=_np(out), q_values=_np(q_values), r=_np(r))
    _dump_net(arrays, "q0", q)
    _dump_dnn(arrays, "im", imitator)
    _save(name, arrays, dict(kind="bcq_model", B=B, S=S, A=A, sizes=list(sizes), thr=thr,
                             imitator_sizes=list(imitator_sizes),
                             imitator_acts=["relu"] * len(imitator_sizes) + ["linear"],
                             state_dict_keys=list(model.state_dict().keys())))


CASES = [
    # seeds chosen so that every filter value stays 1e-4 (relative) away from the threshold and
    # 30-70 % of the actions are dropped (_check_margin)
    (bcq_dqn_case, "dqn_bcq_huber_double", dict(random_masks=True, bcq=0.3, seed=20)),
    (bcq_dqn_case, "dqn_bcq_cpe_mse_single", dict(cpe_metrics=["m1"], loss="mse", double_q=False,
                                                  random_masks=True, bcq=0.3, seed=23,
                                                  temperature=0.5)),
    (bcq_dqn_case, "dqn_bcq_dueling_multistep_boost", dict(dueling=True, sizes=(24, 16),
                                                           multi_steps=3,
                                                           boost={"1": 0.5, "3": -0.25},
                                                           bcq=0.3, seed=23)),
    (bcq_model_case, "bcq_model_forward", dict(seed=25)),
]


def main(only=None):
    for fn, name, kw in CASES:
        if only and name not in only:
            continue
        fn(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
