"""Generate the SAC value-network / CRR golden vectors in tests/golden/ by running the
UNMODIFIED reference SACTrainer (reagent/training/sac_trainer.py) from /root/reference
(build container only; the files are committed because the reference does not travel to the
GPU box).

    python oracle/make_sac_value_golden.py [name ...]

Same recorder pattern as oracle/make_golden.py: torch.randn_like is patched so that the
actor's noise draw is recorded; with a value network each update makes exactly one draw.
Every .npz holds the batch, the initial networks, the draws, the losses of every yield, the
update-0 gradients of every optimizer and the final q1, q2, actor, value and value-target
networks and log_alpha.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import (_NoiseRecorder, _dump_net, _np, _perturb,  # noqa: E402
                                _policy_batch, _save)
from oracle.ref_harness import ref, run_update  # noqa: E402


def sac_value_case(name, *, B=40, S=10, A=3, sizes=(16, 12), acts=("relu", "relu"), twin=True,
                   learn_alpha=True, gamma=0.95, tau=0.05, lr=3e-3, entropy_temperature=0.2,
                   target_entropy=-1.5, uniform_prior=True, crr=None, value_bias=None, seed=0,
                   n_updates=3, perturb=True, both_sides=False):
    """`crr`: CRRWeightFn fields or None.  `value_bias`: the value network's output bias, to
    put the CRR advantages on both sides of a threshold or clamp, which `both_sides` asserts."""
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    actor_mod = ref("reagent.models.actor")
    critic_mod = ref("reagent.models.critic")
    fc_mod = ref("reagent.models.fully_connected_network")
    tr = ref("reagent.training.sac_trainer")
    union = ref("reagent.optimizer.union")
    torch.manual_seed(seed)
    actor = actor_mod.GaussianFullyConnectedActor(S, A, list(sizes), list(acts))
    q1 = critic_mod.FullyConnectedCritic(S, A, list(sizes), list(acts))
    q2 = critic_mod.FullyConnectedCritic(S, A, list(sizes), list(acts)) if twin else None
    value = fc_mod.FloatFeatureFullyConnected(S, 1, list(sizes), list(acts))
    if perturb:
        for m in (actor, q1, q2, value):
            if m is not None:
                _perturb(m)
    if value_bias is not None:
        with torch.no_grad():
            value.fc.dnn[-1][0].bias.fill_(value_bias)
    opt = lambda: union.Optimizer__Union(Adam=union.classes["Adam"](lr=lr))  # noqa: E731
    trainer = tr.SACTrainer(
        actor, q1, q2, value, rl=params.RLParameters(gamma=gamma, target_update_rate=tau),
        q_network_optimizer=opt(), value_network_optimizer=opt(), actor_network_optimizer=opt(),
        alpha_optimizer=opt() if learn_alpha else None, minibatch_size=B,
        entropy_temperature=entropy_temperature, logged_action_uniform_prior=uniform_prior,
        target_entropy=target_entropy,
        crr_config=None if crr is None else tr.CRRWeightFn(**crr))
    keys = set(trainer.state_dict().keys())
    assert not any(k.startswith(("q1_network_target", "q2_network_target")) for k in keys)
    batch, rb = _policy_batch(rlt, B, S, A, seed + 1)
    arrays = {f"batch.{k}": _np(v) for k, v in batch.items()}
    _dump_net(arrays, "actor0", actor)
    _dump_net(arrays, "q1_0", q1)
    if twin:
        _dump_net(arrays, "q2_0", q2)
    _dump_net(arrays, "v0", value)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    all_losses = []
    crr_w = []
    with _NoiseRecorder(seed + 2) as rec:
        for it in range(n_updates):
            cap = {}
            n0 = len(rec.log)
            if crr is not None:
                # the weights this update's actor loss sees: pre-update V, post-critic-update q
                orig = trainer.crr_config.get_weight_from_advantage
                trainer.crr_config.get_weight_from_advantage = \
                    lambda adv, orig=orig: crr_w.append(orig(adv)) or crr_w[-1]
            losses = run_update(trainer, rb, it, opts, capture=cap)
            if crr is not None:
                trainer.crr_config.get_weight_from_advantage = orig
            assert len(rec.log) - n0 == 1, len(rec.log) - n0
            arrays[f"noise{it}.cur"] = _np(rec.log[n0])
            all_losses.append([np.nan if l is None else l for l in losses[:-1]])
            if it == 0:
                for oi, gl in cap.items():
                    for pi, g in enumerate(gl):
                        if g is not None:
                            arrays[f"grad0.opt{oi}.{pi}"] = _np(g)
    if both_sides:
        w = torch.cat([x.reshape(-1) for x in crr_w])
        arrays["crr_weight"] = _np(w)
        if crr.get("exponent_clamp"):
            c = crr["exponent_clamp"]
            assert bool((w >= c).any()) and bool((w < c).any()), "rows on both sides of the clamp"
        else:
            assert bool((w == 1).any()) and bool((w == 0).any()), "rows on both sides"
    arrays["losses"] = np.array(all_losses, dtype=np.float64)
    _dump_net(arrays, "actorN", actor)
    _dump_net(arrays, "q1_N", q1)
    if twin:
        _dump_net(arrays, "q2_N", q2)
    _dump_net(arrays, "vN", value)
    _dump_net(arrays, "vt_N", trainer.value_network_target)
    if learn_alpha:
        arrays["log_alpha_N"] = _np(trainer.log_alpha)
    meta = dict(kind="sac_value", B=B, S=S, A=A, sizes=list(sizes), acts=list(acts), twin=twin,
                learn_alpha=learn_alpha, gamma=gamma, tau=tau, lr=lr,
                entropy_temperature=entropy_temperature, target_entropy=target_entropy,
                uniform_prior=uniform_prior, crr=crr, n_updates=n_updates,
                state_dict_keys=sorted(keys))
    _save(name, arrays, meta)


# The reference's Pendulum configurations (reagent/gym/tests/configs/pendulum/
# sac_pendulum_online.yaml, continuous_crr_pendulum_online.yaml) as the reference SAC manager
# wires them (reagent/model_managers/actor_critic/sac.py:80-113): S 3, A 1, minibatch 256,
# [64, 64] leaky_relu actor, critics and value network, gamma 0.99, tau 0.005,
# entropy_temperature 0.3, Adam(1e-3) everywhere (the CRR config leaves alpha_optimizer at its
# default, Adam(1e-3)), target_entropy -1, logged_action_uniform_prior True.
PENDULUM = dict(B=256, S=3, A=1, sizes=(64, 64), acts=("leaky_relu", "leaky_relu"), twin=True,
                learn_alpha=True, gamma=0.99, tau=0.005, lr=1e-3, entropy_temperature=0.3,
                target_entropy=-1.0, uniform_prior=True, n_updates=5, perturb=False)


def main(only=None):
    cases = [
        ("sac_value_twin_alpha", {}),
        # a fixed alpha: with a learnable one the reference's value target is float64 (log_alpha
        # is) and its mse_loss backward raises "Found dtype Double but expected Float"
        ("sac_value_single_prior", dict(twin=False, uniform_prior=False, learn_alpha=False,
                                        entropy_temperature=0.35, seed=3,
                                        acts=("tanh", "leaky_relu"))),
        ("sac_value_fixed_alpha_odd", dict(learn_alpha=False, B=37, S=7, A=2, sizes=(10,),
                                           acts=("relu",), gamma=0.0, seed=5)),
        ("sac_crr_exponent", dict(crr=dict(exponent_beta=1.0, exponent_clamp=20.0),
                                  value_bias=-3.0, seed=7, both_sides=True)),
        ("sac_crr_indicator", dict(crr=dict(indicator_fn_threshold=0.05), seed=9,
                                   both_sides=True)),
        ("sac_pendulum_manager", dict(PENDULUM, seed=11)),
        ("sac_crr_pendulum_manager", dict(PENDULUM, crr=dict(exponent_beta=1.0,
                                                             exponent_clamp=20.0), seed=13)),
    ]
    for name, kw in cases:
        if only and name not in only:
            continue
        sac_value_case(name, **kw)


if __name__ == "__main__":
    main(sys.argv[1:] or None)
