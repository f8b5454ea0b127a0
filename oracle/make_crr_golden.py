"""Generate the discrete-CRR golden vectors in tests/golden/ by running the UNMODIFIED reference
DiscreteCRRTrainer (reagent/training/discrete_crr_trainer.py) through oracle/ref_harness.py.
Needs the reference checkout (build container only); the files are committed.

    python oracle/make_crr_golden.py            # regenerate every case
    python oracle/make_crr_golden.py NAME ...   # only the named ones

Every update runs on the same batch.  torch.distributions.Normal.sample is wrapped while the
trainer runs, so that the two exploration-noise draws of an update (the actor's forward on
next_state, then on state; both happen on every batch, also when the actor step is skipped) are
recorded as the reference made them.  Each file holds
  batch.*                       state, next_state, action, reward, not_terminal,
                                action_probability, possible_next_actions_mask[, metrics]
  <net>0.W*/b*, <net>N.W*/b*    actor, actor_t, q1, q1_t[, q2, q2_t, r, c, ct] before / after
  noise{t}.next / noise{t}.cur  the draws of update t (absent without exploration_variance)
  losses                        [n_updates, n_optimizers - 1], NaN for a `None` yield
  grad0.opt{i}.{p}              update-0 gradients of optimizer i
  weight0                       the actor weights of update 0
and the structure in the metadata (`optimizers`: which network each optimizer steps).
`crr_cartpole_manager` is the reference's CartPole configuration (reagent/gym/tests/configs/
cartpole/discrete_crr_cartpole_online.yaml) with the networks DiscreteCRR.build_trainer gives it
(reagent/model_managers/discrete/discrete_crr.py:104-179): [1024, 1024] actor and twin critics.
Those are too large to commit, so its initial parameters come from crr_oracle.seeded_like and
its gradients and final parameters are stored as crr_oracle.digest samples.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.crr_oracle import digest, seeded_like  # noqa: E402
from oracle.make_golden import _dump_net, _fc_params, _np, _perturb, _save  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402


class _NormalSampleRecorder:
    def __enter__(self):
        self.log = []
        self._orig = torch.distributions.Normal.sample
        rec = self

        def sample(dist, sample_shape=torch.Size()):
            out = rec._orig(dist, sample_shape)
            rec.log.append(out.clone())
            return out

        torch.distributions.Normal.sample = sample
        return self

    def __exit__(self, *exc):
        torch.distributions.Normal.sample = self._orig


def _flat_params(net):
    return [p for pair in _fc_params(net) for p in pair]


def crr_case(name, *, B=40, S=9, A=4, sizes=(16, 12), acts=("relu", "relu"), twin=True,
             dueling=False, use_target_actor=False, delayed_policy_update=1, beta=1.0,
             entropy_coeff=0.0, clip_limit=10.0, max_weight=20.0, exploration_variance=None,
             actor_scale=None, cpe_metrics=None, boost=None, optimizer="Adam", opt_kw=None,
             gamma=0.97, tau=0.05, temperature=0.1, lr=3e-3, seed=0, n_updates=3, probs=None,
             compact=False, check=None):
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    actor_mod = ref("reagent.models.actor")
    dqn_mod = ref("reagent.models.dqn")
    tr = ref("reagent.training.discrete_crr_trainer")
    union = ref("reagent.optimizer.union")
    torch.manual_seed(seed)
    sizes, acts = list(sizes), list(acts)

    def critic():
        if dueling:
            duel = ref("reagent.models.dueling_q_network")
            return duel.DuelingQNetwork.make_fully_connected(S, A, sizes, acts)
        return dqn_mod.FullyConnectedDQN(S, A, sizes, acts)

    actor = actor_mod.FullyConnectedActor(S, A, sizes, acts,
                                          exploration_variance=exploration_variance)
    q1 = critic()
    q2 = critic() if twin else None
    cpe = cpe_metrics is not None
    reward_net = qcpe = None
    if cpe:
        n_out = (len(cpe_metrics) + 1) * A
        reward_net = dqn_mod.FullyConnectedDQN(S, n_out, sizes, acts)
        qcpe = dqn_mod.FullyConnectedDQN(S, n_out, sizes, acts)
    sources = [("actor", actor), ("q1", q1), ("q2", q2), ("r", reward_net), ("c", qcpe)]
    sources = [(k, m) for k, m in sources if m is not None]
    with torch.no_grad():
        for i, (_, m) in enumerate(sources):
            if compact:
                for p, v in zip(_flat_params(m), seeded_like(_flat_params(m), seed + 100 + i)):
                    p.copy_(v)
            else:
                _perturb(m)
        if actor_scale is not None:  # drive tanh towards +-1 so that the noise clamp binds
            w, b = _fc_params(actor)[-1]
            w.mul_(actor_scale)
            b.mul_(actor_scale)
    targets = {"actor_t": actor.get_target_network(), "q1_t": q1.get_target_network()}
    if twin:
        targets["q2_t"] = q2.get_target_network()
    if cpe:
        targets["ct"] = qcpe.get_target_network()
    if not compact:  # targets that differ from their sources, so that the soft update shows
        with torch.no_grad():
            for m in targets.values():
                for w, b in _fc_params(m):
                    w.add_(torch.randn_like(w) * 0.05)
                    b.add_(torch.randn_like(b) * 0.05)
    actions = [str(i) for i in range(A)]
    opt = lambda: union.Optimizer__Union(**{optimizer: union.classes[optimizer](  # noqa: E731
        lr=lr, **(opt_kw or {}))})
    trainer = tr.DiscreteCRRTrainer(
        actor_network=actor, actor_network_target=targets["actor_t"], q1_network=q1,
        q1_network_target=targets["q1_t"], reward_network=reward_net, q2_network=q2,
        q2_network_target=targets.get("q2_t"), q_network_cpe=qcpe,
        q_network_cpe_target=targets.get("ct"),
        metrics_to_score=list(cpe_metrics) if cpe else None,
        evaluation=params.EvaluationParameters(calc_cpe_in_training=cpe),
        rl=params.RLParameters(gamma=gamma, target_update_rate=tau, reward_boost=boost,
                               temperature=temperature),
        double_q_learning=twin, q_network_optimizer=opt(), actor_network_optimizer=opt(),
        use_target_actor=use_target_actor, actions=actions,
        delayed_policy_update=delayed_policy_update, beta=beta, entropy_coeff=entropy_coeff,
        clip_limit=clip_limit, max_weight=max_weight)
    gen = torch.Generator().manual_seed(seed + 1)
    act_idx = torch.randint(A, (B,), generator=gen)
    batch = dict(
        state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
        reward=torch.randn(B, 1, generator=gen),
        not_terminal=(torch.rand(B, 1, generator=gen) > 0.2).float(),
        action=torch.nn.functional.one_hot(act_idx, A).float(),
        possible_next_actions_mask=torch.ones(B, A),
        action_probability=(torch.rand(B, 1, generator=gen) * 0.8 + 0.1) if probs is None
        else torch.tensor(probs, dtype=torch.float32)[torch.arange(B) % len(probs)].view(B, 1))
    if cpe:
        batch["metrics"] = torch.randn(B, len(cpe_metrics), generator=gen)
    rbatch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(batch["state"]), next_state=rlt.FeatureData(batch["next_state"]),
        reward=batch["reward"], time_diff=torch.ones(B, 1), step=None,
        not_terminal=batch["not_terminal"], action=batch["action"],
        next_action=torch.zeros(B, A), possible_actions_mask=torch.ones(B, A),
        possible_next_actions_mask=batch["possible_next_actions_mask"],
        extras=rlt.ExtraData(action_probability=batch["action_probability"],
                             metrics=batch.get("metrics")))
    arrays = {f"batch.{k}": _np(v) for k, v in batch.items()}
    nets = dict(sources, **targets)
    if not compact:
        for k, m in nets.items():
            _dump_net(arrays, k + "0", m)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    owner = {id(p): k for k, m in nets.items() for p in m.parameters()}
    structure = [owner[id(o.param_groups[0]["params"][0])] for o in opts[:-1]]
    # the soft update's targets, in order (its params are targets then sources)
    su = opts[-1].param_groups[0]["params"]
    su_targets = list(dict.fromkeys(owner[id(p)] for p in su[:len(su) // 2]))
    weights = []
    orig_loss = trainer.compute_actor_loss

    def spy(batch_idx, action, logged_action_probs, all_q_values, all_action_scores):
        if batch_idx % delayed_policy_update == 0:
            v = (all_q_values * torch.softmax(all_action_scores, 1)).sum(1, keepdim=True)
            adv = ((all_q_values - v) * action).sum(1, keepdim=True)
            weights.append(torch.clamp(((1 / beta) * adv).exp(), 0, max_weight).detach())
            if entropy_coeff > 0:
                pi_t = (torch.softmax(all_action_scores, 1) * action).sum(1, keepdim=True)
                weights.append((pi_t / logged_action_probs.view(-1, 1)).detach())
        return orig_loss(batch_idx, action, logged_action_probs, all_q_values, all_action_scores)

    trainer.compute_actor_loss = spy
    all_losses = []
    with _NormalSampleRecorder() as rec:
        for it in range(n_updates):
            before = {k: [p.detach().clone() for p in m.parameters()] for k, m in targets.items()}
            cap, n0 = {}, len(rec.log)
            losses = run_update(trainer, rbatch, it, opts, capture=cap)
            draws = rec.log[n0:]
            assert len(draws) == (0 if exploration_variance is None else 2), len(draws)
            if draws:
                arrays[f"noise{it}.next"], arrays[f"noise{it}.cur"] = _np(draws[0]), _np(draws[1])
            all_losses.append([np.nan if l is None else l for l in losses[:-1]])
            if it % delayed_policy_update != 0:
                # the actor's yield was None, and the soft update still moved every target
                assert losses[structure.index("actor")] is None
                for k, m in targets.items():
                    assert any(not torch.equal(a, b) for a, b in zip(before[k], m.parameters())), k
            if it == 0:
                for oi, gl in cap.items():
                    for pi, g in enumerate(gl):
                        if g is not None:
                            arrays[f"grad0.opt{oi}.{pi}"] = _np(digest(g)) if compact else _np(g)
    arrays["weight0"] = _np(weights[0].view(-1))
    if check is not None:
        check(weights, [arrays.get(f"noise{t}.cur") for t in range(n_updates)], actor, batch)
    arrays["losses"] = np.array(all_losses, dtype=np.float64)
    for k, m in nets.items():
        if compact:
            for i, p in enumerate(_flat_params(m)):
                arrays[f"{k}N.digest{i}"] = _np(digest(p))
        else:
            _dump_net(arrays, k + "N", m)
    meta = dict(kind="crr", B=B, S=S, A=A, sizes=sizes, acts=acts, twin=twin, dueling=dueling,
                use_target_actor=use_target_actor, delayed_policy_update=delayed_policy_update,
                beta=beta, entropy_coeff=entropy_coeff, clip_limit=clip_limit,
                max_weight=max_weight, exploration_variance=exploration_variance,
                cpe_metrics=cpe_metrics, boost=boost, optimizer=optimizer, opt_kw=opt_kw or {},
                gamma=gamma, tau=tau, temperature=temperature, lr=lr, seed=seed,
                n_updates=n_updates, compact=compact, optimizers=structure,
                soft_update_targets=su_targets, n_yields=len(opts))
    _save(name, arrays, meta)


def _check_entropy_clip(weights, noises, actor, batch):
    w, ratio = weights[0], weights[1]
    assert bool((w >= 1.0).any()) and bool((w < 1.0).any()), "rows on both sides of max_weight"
    assert bool((ratio < 1e-4).any()) and bool((ratio > 1.2).any()), "both ends of the ratio clip"
    assert bool(((ratio > 1e-4) & (ratio < 1.2)).any()), "unclipped ratios"


def _check_saturated(weights, noises, actor, batch):
    rlt = ref("reagent.core.types")
    with torch.no_grad():
        raw = actor.fc(batch["state"]) + torch.from_numpy(noises[-1])
    out = (raw.abs() > 1).float().mean()
    assert 0.05 < float(out) < 0.95, f"clamp active on {float(out):.2f} of the entries"
    del rlt


CASES = [
    ("crr_twin_default", {}),
    ("crr_single_target_actor", dict(twin=False, use_target_actor=True, seed=2,
                                     acts=("tanh", "leaky_relu"))),
    ("crr_dueling_delayed", dict(dueling=True, delayed_policy_update=2, n_updates=4, seed=4,
                                 sizes=(16, 12))),
    ("crr_entropy_clip", dict(entropy_coeff=0.3, clip_limit=1.2, max_weight=1.0, beta=0.5,
                              probs=[0.05, 0.5, 1e5, 0.9], seed=6, check=_check_entropy_clip)),
    ("crr_noise_saturated", dict(exploration_variance=0.5, actor_scale=6.0, seed=8,
                                 check=_check_saturated)),
    ("crr_cpe_boost", dict(cpe_metrics=["m0"], boost={"1": 0.7, "3": -0.4}, seed=10)),
    ("crr_adamw_amsgrad", dict(optimizer="AdamW", opt_kw=dict(amsgrad=True, weight_decay=0.01),
                               seed=12)),
    ("crr_odd_dims", dict(B=37, S=7, A=3, sizes=(10, 6), seed=14, exploration_variance=0.05)),
    # discrete_crr_cartpole_online.yaml: gamma 0.99, tau 0.2, temperature 0.1, twin critics,
    # delayed_policy_update 1, Adam(1e-3), [1024, 1024] relu, exploration_variance 1e-7,
    # FullyConnected critics, minibatch 256 on CartPole (S 4, A 2), no CPE in training
    ("crr_cartpole_manager", dict(B=256, S=4, A=2, sizes=(1024, 1024), gamma=0.99, tau=0.2,
                                  temperature=0.1, lr=1e-3, exploration_variance=1e-7, seed=16,
                                  compact=True)),
]


def main(only=None):
    for name, kw in CASES:
        if only and name not in only:
            continue
        crr_case(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
