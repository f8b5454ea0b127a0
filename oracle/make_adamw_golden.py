"""Golden vectors for torch.optim.AdamW (with and without AMSGrad) under the reference's own
trainers, written to tests/golden/.  Like make_golden.py this runs the UNMODIFIED reference
through oracle/ref_harness.py; the reference's `AdamW` config builds torch.optim.AdamW.

    python oracle/make_adamw_golden.py            # regenerate every case
    python oracle/make_adamw_golden.py NAME ...   # only the named cases

Each case runs N_UPDATES consecutive updates, each on its own seeded batch, so that the decay
and the AMSGrad maximum build up.  Update k's batch is stored under `batch{k}.`; the losses of
every update and the parameters after the last one are stored as in make_golden.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle.make_golden import (_NoiseRecorder, _dump_net, _fc_params, _np, _perturb,  # noqa: E402
                                _policy_batch, _save)
from oracle.ref_harness import ref, run_update  # noqa: E402

N_UPDATES = 5


def _adamw(lr, weight_decay, amsgrad):
    union = ref("reagent.optimizer.union")
    return union.Optimizer__Union(AdamW=union.classes["AdamW"](
        lr=lr, weight_decay=weight_decay, amsgrad=amsgrad))


def _perturb_target(module):
    with torch.no_grad():
        for w, b in _fc_params(module):
            w.add_(torch.randn_like(w) * 0.05)
            b.add_(torch.randn_like(b) * 0.05)


def _discrete_batch(rlt, B, S, A, gen, round_rewards=False):
    act_idx = torch.randint(A, (B,), generator=gen)
    nact_idx = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.2).float()
    reward = torch.randn(B, 1, generator=gen)
    if round_rewards:  # C51: rewards on the support points as well as between them
        reward[: B // 4] = torch.round(reward[: B // 4])
    batch = dict(state=torch.randn(B, S, generator=gen),
                 next_state=torch.randn(B, S, generator=gen), reward=reward,
                 time_diff=torch.ones(B, 1), step=torch.ones(B, 1, dtype=torch.int64),
                 not_terminal=nt, action=torch.nn.functional.one_hot(act_idx, A).float(),
                 next_action=torch.nn.functional.one_hot(nact_idx, A).float() * nt,
                 possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    rbatch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(batch["state"]), next_state=rlt.FeatureData(batch["next_state"]),
        reward=batch["reward"], time_diff=batch["time_diff"], step=None, not_terminal=nt,
        action=batch["action"], next_action=batch["next_action"],
        possible_actions_mask=batch["possible_actions_mask"],
        possible_next_actions_mask=batch["possible_next_actions_mask"],
        extras=rlt.ExtraData(action_probability=torch.ones(B, 1)))
    return batch, rbatch


def _run_discrete(trainer, rlt, arrays, B, S, A, seed, round_rewards=False):
    gen = torch.Generator().manual_seed(seed + 1)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    assert type(opts[0]) is torch.optim.AdamW, type(opts[0])
    losses = []
    for it in range(N_UPDATES):
        batch, rbatch = _discrete_batch(rlt, B, S, A, gen, round_rewards)
        arrays.update({f"batch{it}.{k}": _np(v) for k, v in batch.items()})
        losses.append(run_update(trainer, rbatch, it, opts)[0])
    arrays["losses"] = np.array(losses, dtype=np.float64)


def _meta(lr, weight_decay, amsgrad, **kw):
    return dict(kw, lr=lr, weight_decay=weight_decay, amsgrad=amsgrad, optimizer="AdamW",
                n_updates=N_UPDATES, multi_steps=None, time_diff=False, boost=None,
                double_q=True, maxq=True)


def qrdqn_case(name, *, B, S, A, N, sizes, acts, gamma, tau, lr, weight_decay, amsgrad, seed):
    """DuelingQuantile network, as the DiscreteQRDQN manager builds it."""
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    duel = ref("reagent.models.dueling_q_network")
    tr = ref("reagent.training.qrdqn_trainer")
    torch.manual_seed(seed)
    q = duel.DuelingQNetwork.make_fully_connected(S, A, list(sizes), list(acts), num_atoms=N)
    with torch.no_grad():  # biases are 0 at init in the reference: exercise the bias paths
        for _, b in _fc_params(q):
            b.normal_(0, 0.1)
    qt = q.get_target_network()
    _perturb_target(qt)
    trainer = tr.QRDQNTrainer(
        q, qt, actions=[str(i) for i in range(A)],
        rl=params.RLParameters(gamma=gamma, target_update_rate=tau, maxq_learning=True),
        double_q_learning=True, num_atoms=N, minibatch_size=B,
        optimizer=_adamw(lr, weight_decay, amsgrad),
        evaluation=params.EvaluationParameters(calc_cpe_in_training=False))
    arrays = {}
    _dump_net(arrays, "q0", q)
    _dump_net(arrays, "qt0", qt)
    _run_discrete(trainer, rlt, arrays, B, S, A, seed)
    _dump_net(arrays, "qN", q)
    _dump_net(arrays, "qtN", qt)
    _save(name, arrays, _meta(lr, weight_decay, amsgrad, kind="qrdqn", B=B, S=S, A=A, N=N,
                              sizes=list(sizes), acts=list(acts), gamma=gamma, tau=tau,
                              dueling=True))


def c51_case(name, *, B, S, A, N, qmin, qmax, sizes, acts, gamma, tau, lr, weight_decay,
             amsgrad, seed):
    """Categorical network, as the DiscreteC51DQN manager builds it."""
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    dqn_mod = ref("reagent.models.dqn")
    cat = ref("reagent.models.categorical_dqn")
    tr = ref("reagent.training.c51_trainer")
    torch.manual_seed(seed)
    # reagent/net_builder/categorical_dqn/categorical.py:29-49
    dist = dqn_mod.FullyConnectedDQN(S, A, list(sizes), list(acts), num_atoms=N,
                                     use_batch_norm=False, dropout_ratio=0.0)
    with torch.no_grad():
        for _, b in _fc_params(dist):
            b.normal_(0, 0.1)
    q = cat.CategoricalDQN(dist, qmin=qmin, qmax=qmax, num_atoms=N)
    qt = q.get_target_network()
    _perturb_target(qt.distributional_network)
    trainer = tr.C51Trainer(
        q, qt, actions=[str(i) for i in range(A)],
        rl=params.RLParameters(gamma=gamma, target_update_rate=tau, maxq_learning=True),
        double_q_learning=True, minibatch_size=B, num_atoms=N, qmin=qmin, qmax=qmax,
        optimizer=_adamw(lr, weight_decay, amsgrad))
    arrays = {}
    _dump_net(arrays, "q0", q.distributional_network)
    _dump_net(arrays, "qt0", qt.distributional_network)
    _run_discrete(trainer, rlt, arrays, B, S, A, seed, round_rewards=True)
    _dump_net(arrays, "qN", q.distributional_network)
    _dump_net(arrays, "qtN", qt.distributional_network)
    _save(name, arrays, _meta(lr, weight_decay, amsgrad, kind="c51", B=B, S=S, A=A, N=N,
                              qmin=qmin, qmax=qmax, sizes=list(sizes), acts=list(acts),
                              gamma=gamma, tau=tau))


def dqn_case(name, *, B, S, A, sizes, acts, gamma, tau, lr, weight_decay, amsgrad, seed):
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    dqn_mod = ref("reagent.models.dqn")
    tr = ref("reagent.training.dqn_trainer")
    torch.manual_seed(seed)
    q = dqn_mod.FullyConnectedDQN(S, A, list(sizes), list(acts))
    with torch.no_grad():
        for _, b in _fc_params(q):
            b.normal_(0, 0.1)
    qt = q.get_target_network()
    _perturb_target(qt)
    trainer = tr.DQNTrainer(
        q, qt, None, None, None, actions=[str(i) for i in range(A)],
        rl=params.RLParameters(gamma=gamma, target_update_rate=tau, q_network_loss="mse"),
        double_q_learning=True, minibatch_size=B, optimizer=_adamw(lr, weight_decay, amsgrad),
        evaluation=params.EvaluationParameters(calc_cpe_in_training=False))
    arrays = {}
    _dump_net(arrays, "q0", q)
    _dump_net(arrays, "qt0", qt)
    _run_discrete(trainer, rlt, arrays, B, S, A, seed)
    _dump_net(arrays, "qN", q)
    _dump_net(arrays, "qtN", qt)
    _save(name, arrays, _meta(lr, weight_decay, amsgrad, kind="dqn", B=B, S=S, A=A,
                              sizes=list(sizes), acts=list(acts), loss="mse", gamma=gamma,
                              tau=tau, dueling=False, cpe_metrics=None))


def sac_case(name, *, B, S, A, sizes, acts, gamma, tau, lr, weight_decay, amsgrad,
             entropy_temperature, target_entropy, seed):
    """AdamW on all four optimizers, including the stand-alone log_alpha."""
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    actor_mod = ref("reagent.models.actor")
    critic_mod = ref("reagent.models.critic")
    tr = ref("reagent.training.sac_trainer")
    torch.manual_seed(seed)
    actor = actor_mod.GaussianFullyConnectedActor(S, A, list(sizes), list(acts))
    q1 = critic_mod.FullyConnectedCritic(S, A, list(sizes), list(acts))
    q2 = critic_mod.FullyConnectedCritic(S, A, list(sizes), list(acts))
    for m in (actor, q1, q2):
        _perturb(m)
    opt = lambda: _adamw(lr, weight_decay, amsgrad)  # noqa: E731
    trainer = tr.SACTrainer(
        actor, q1, q2, rl=params.RLParameters(gamma=gamma, target_update_rate=tau),
        q_network_optimizer=opt(), actor_network_optimizer=opt(), alpha_optimizer=opt(),
        minibatch_size=B, entropy_temperature=entropy_temperature,
        target_entropy=target_entropy)
    arrays = {}
    _dump_net(arrays, "actor0", actor)
    _dump_net(arrays, "q1_0", q1)
    _dump_net(arrays, "q2_0", q2)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    assert all(type(o) is torch.optim.AdamW for o in opts[:-1]), opts
    all_losses = []
    with _NoiseRecorder(seed + 2) as rec:
        for it in range(N_UPDATES):
            batch, rb = _policy_batch(rlt, B, S, A, seed + 10 + it)
            arrays.update({f"batch{it}.{k}": _np(v) for k, v in batch.items()})
            n0 = len(rec.log)
            losses = run_update(trainer, rb, it, opts)
            assert len(rec.log) - n0 == 2, len(rec.log) - n0
            arrays[f"noise{it}.next"] = _np(rec.log[n0])
            arrays[f"noise{it}.cur"] = _np(rec.log[n0 + 1])
            all_losses.append(losses[:-1])
    arrays["losses"] = np.array(all_losses, dtype=np.float64)
    _dump_net(arrays, "actorN", actor)
    _dump_net(arrays, "q1_N", q1)
    _dump_net(arrays, "q1t_N", trainer.q1_network_target)
    _dump_net(arrays, "q2_N", q2)
    _dump_net(arrays, "q2t_N", trainer.q2_network_target)
    arrays["log_alpha_N"] = _np(trainer.log_alpha)
    _save(name, arrays, dict(kind="sac", B=B, S=S, A=A, sizes=list(sizes), acts=list(acts),
                             twin=True, learn_alpha=True, gamma=gamma, tau=tau, lr=lr,
                             weight_decay=weight_decay, amsgrad=amsgrad, optimizer="AdamW",
                             entropy_temperature=entropy_temperature,
                             target_entropy=target_entropy, backprop=True,
                             n_updates=N_UPDATES))


CASES = {
    # reagent/gym/tests/configs/cartpole/discrete_qr_cartpole_online.yaml
    "qrdqn_adamw_amsgrad_cartpole": (qrdqn_case, dict(
        B=512, S=4, A=2, N=11, sizes=(64, 64), acts=("leaky_relu", "leaky_relu"), gamma=0.9,
        tau=0.05, lr=1e-3, weight_decay=0.01, amsgrad=True, seed=0)),
    # reagent/gym/tests/configs/cartpole/discrete_c51_cartpole_online.yaml
    "c51_adamw_amsgrad_cartpole": (c51_case, dict(
        B=512, S=4, A=2, N=21, qmin=0.0, qmax=40.0, sizes=(64, 64),
        acts=("leaky_relu", "leaky_relu"), gamma=0.9, tau=0.05, lr=1e-3, weight_decay=0.01,
        amsgrad=True, seed=1)),
    # reagent/gym/tests/configs/sparse/discrete_dqn_changing_arms_online.yaml: AdamW(lr=0.005),
    # decay only
    "dqn_adamw_decay": (dqn_case, dict(
        B=64, S=12, A=5, sizes=(24, 20), acts=("relu", "relu"), gamma=0.97, tau=0.05, lr=5e-3,
        weight_decay=0.01, amsgrad=False, seed=2)),
    "sac_adamw_amsgrad": (sac_case, dict(
        B=40, S=10, A=3, sizes=(16, 12), acts=("relu", "relu"), gamma=0.95, tau=0.05, lr=3e-3,
        weight_decay=0.01, amsgrad=True, entropy_temperature=0.2, target_entropy=-1.5,
        seed=3)),
}


def main(only=None):
    for name, (fn, kw) in CASES.items():
        if not only or name in only:
            fn(name, **kw)


if __name__ == "__main__":
    main(sys.argv[1:])
