"""Generate the policy-gradient golden vectors in tests/golden/ by running the UNMODIFIED
reference ReinforceTrainer and PPOTrainer (reagent/training/reinforce_trainer.py,
ppo_trainer.py) through oracle/ref_harness.py.  Needs the reference checkout (build container
only); the files are committed.

    python oracle/make_pg_golden.py            # regenerate every case
    python oracle/make_pg_golden.py NAME ...   # only the named ones

REINFORCE runs one trajectory per update under ref_harness.run_update.  PPO is manually
optimized: its `training_step` is called once per trajectory, with three shims set on the
instance here -- `optimizers()` returns the one list of configure_optimizers(),
`manual_backward(loss)` is `loss.backward()`, the reporter records what `_update_model`
reports -- and `logger` None, so the logger-only `_eval_metrics` does not run.  Each file holds
  traj{k}.*                   state, action, reward, log_prob[, possible_actions_mask,
                              next_state, not_terminal] of trajectory k
  policy0.* / value0.*        the networks before the first update
  policy{u}.* / value{u}.*    after update u (REINFORCE: batch u; PPO: update_model call u)
  dret{i}                     the i-th output of the reference's discounted_returns
  adv{i}                      PPO: the i-th output of _compute_advantage
  losses                      [n minibatches, n optimizers] (value loss first)
  grad0.opt{i}.{p}            the gradients of the first minibatch
  perm{u}.{e}                 PPO: the torch.randperm of update u, epoch e
The CartPole cases wire the networks the reference managers build for
reagent/gym/tests/configs/cartpole/discrete_{reinforce,ppo}_cartpole_online.yaml
(FullyConnected [64] / [32, 32] leaky_relu on S 4, A 2) with the configurations' parameters.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import _dump_net, _np, _perturb, _save  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402


class _Recorder:
    """Records every output of a module-level function while installed."""

    def __init__(self, module, name):
        self.module, self.name, self.log = module, name, []

    def __enter__(self):
        self.orig = getattr(self.module, self.name)

        def wrapped(*a, **k):
            out = self.orig(*a, **k)
            self.log.append(out.detach().clone())
            return out

        setattr(self.module, self.name, wrapped)
        return self

    def __exit__(self, *exc):
        setattr(self.module, self.name, self.orig)


class _Reporter:
    """What _update_model reports: [value_net_loss,] ppo_loss per minibatch."""

    def __init__(self, with_value: bool):
        self.with_value, self.losses = with_value, []

    def log(self, ppo_loss, value_net_loss):
        self.losses.append(([float(value_net_loss)] if self.with_value else []) + [float(ppo_loss)])


def _trajectories(lengths, S, A, seed, *, masked=False, next_state=False, not_terminal=None,
                  constant=(), policy=None, temperature=1.0, ratio_noise=0.0):
    """Random trajectories; log_prob is the current policy's log-probability of the logged
    action plus N(0, ratio_noise) (so PPO ratios land on both sides of the clip), or random."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for k, T in enumerate(lengths):
        mask = None
        if masked:
            mask = (torch.rand(T, A, generator=g) > 0.3).float()
            mask[torch.arange(T), torch.randint(A, (T,), generator=g)] = 1.0
        probs = torch.ones(T, A) if mask is None else mask
        act = torch.multinomial(probs, 1, generator=g).view(-1)
        d = dict(state=torch.randn(T, S, generator=g),
                 action=torch.nn.functional.one_hot(act, A).float(),
                 reward=torch.randn(T, generator=g) * 2.0)
        if k in constant:
            d["reward"] = torch.ones(T)
        if policy is not None:
            with torch.no_grad():
                sc = policy(ref("reagent.core.types").FeatureData(d["state"]))
                if mask is not None:
                    sc = sc + (-1e10) * (1 - mask)
                lp = torch.distributions.Categorical(logits=sc / temperature).log_prob(act)
            d["log_prob"] = lp + torch.randn(T, generator=g) * ratio_noise
        else:
            d["log_prob"] = torch.log(torch.rand(T, generator=g) * 0.9 + 0.05)
        if mask is not None:
            d["possible_actions_mask"] = mask
        if next_state:
            d["next_state"] = torch.randn(T, S, generator=g)
        if not_terminal is not None:
            nt = (torch.rand(T, generator=g) > 0.1).float()
            nt[-1] = not_terminal[k]
            d["not_terminal"] = nt
        out.append(d)
    return out


def _rlt_traj(rlt, d):
    return rlt.PolicyGradientInput(
        state=rlt.FeatureData(d["state"]), action=d["action"], reward=d["reward"],
        log_prob=d["log_prob"], possible_actions_mask=d.get("possible_actions_mask"),
        next_state=rlt.FeatureData(d["next_state"]) if "next_state" in d else None,
        not_terminal=d.get("not_terminal"))


def _nets(S, A, sizes, acts, dueling, value_sizes, seed):
    dqn = ref("reagent.models.dqn")
    torch.manual_seed(seed)
    if dueling:
        duel = ref("reagent.models.dueling_q_network")
        policy = duel.DuelingQNetwork.make_fully_connected(S, A, list(sizes), list(acts))
    else:
        policy = dqn.FullyConnectedDQN(S, A, list(sizes), list(acts))
    _perturb(policy)
    value = None
    if value_sizes is not None:
        fc = ref("reagent.models.fully_connected_network")
        value = fc.FloatFeatureFullyConnected(S, 1, list(value_sizes), ["relu"] * len(value_sizes))
        _perturb(value)
    return policy, value


def _opt(union, lr, wd):
    return union.Optimizer__Union(Adam=union.classes["Adam"](lr=lr, weight_decay=wd))


def _grad_recorder(opts, arrays):
    """Wrap each optimizer's step so that the gradients of the first minibatch are stored."""
    seen = set()
    for i, o in enumerate(opts):
        orig = o.step

        def step(*a, _i=i, _o=o, _orig=orig, **k):
            if _i not in seen:
                seen.add(_i)
                for pi, p in enumerate(p for g in _o.param_groups for p in g["params"]):
                    if p.grad is not None:
                        arrays[f"grad0.opt{_i}.{pi}"] = _np(p.grad).copy()
            return _orig(*a, **k)

        o.step = step


def _run_untoggled(trainer, batch, batch_idx, opts, capture):
    """run_update without Lightning's optimizer toggling.  With a value net the reference's
    generator runs the policy forward before its first yield, while the value optimizer is
    toggled on and the policy's parameters do not require grad, so under the toggle its policy
    loss has no graph.  The two losses depend on disjoint parameters (the advantage is
    detached), so each optimizer steps on its own loss in yield order."""
    gen = trainer.train_step_gen(batch, batch_idx)
    losses = []
    for i, opt in enumerate(opts):
        loss = next(gen)
        opt.zero_grad()
        loss.backward()
        capture[i] = [p.grad.detach().clone() for g in opt.param_groups for p in g["params"]]
        opt.step()
        losses.append(float(loss.detach()))
    return losses


def reinforce_case(name, *, lengths, S=4, A=2, sizes=(64,), acts=("leaky_relu",), dueling=False,
                   value_sizes=None, gamma=0.0, lr=1e-3, wd=0.0, off_policy=False,
                   reward_clip=1e6, clip_param=1e6, normalize=True, subtract_mean=True,
                   offset_clamp_min=False, temperature=1.0, masked=False, constant=(), seed=0):
    rlt = ref("reagent.core.types")
    union = ref("reagent.optimizer.union")
    tr = ref("reagent.training.reinforce_trainer")
    pol_mod = ref("reagent.gym.policies.policy")
    samp = ref("reagent.gym.policies.samplers.discrete_sampler")
    policy, value = _nets(S, A, sizes, acts, dueling, value_sizes, seed)
    trajs = _trajectories(lengths, S, A, seed + 1, masked=masked, constant=constant)
    trainer = tr.ReinforceTrainer(
        policy=pol_mod.Policy(scorer=policy, sampler=samp.SoftmaxActionSampler(temperature)),
        gamma=gamma, optimizer=_opt(union, lr, wd), optimizer_value_net=_opt(union, lr, wd),
        actions=[str(i) for i in range(A)], off_policy=off_policy, reward_clip=reward_clip,
        clip_param=clip_param, normalize=normalize, subtract_mean=subtract_mean,
        offset_clamp_min=offset_clamp_min, value_net=value)
    arrays = {}
    for k, d in enumerate(trajs):
        for f, v in d.items():
            arrays[f"traj{k}.{f}"] = _np(v)
    _dump_net(arrays, "policy0", policy)
    if value is not None:
        _dump_net(arrays, "value0", value)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    all_losses = []
    with _Recorder(tr, "discounted_returns") as rec:
        for u, d in enumerate(trajs):
            cap = {}
            run = run_update if value is None else _run_untoggled
            all_losses.append(run(trainer, _rlt_traj(rlt, d), u, opts, capture=cap))
            if u == 0:
                for oi, gl in cap.items():
                    for pi, gr in enumerate(gl):
                        arrays[f"grad0.opt{oi}.{pi}"] = _np(gr)
            _dump_net(arrays, f"policy{u + 1}", policy)
            if value is not None:
                _dump_net(arrays, f"value{u + 1}", value)
    for i, r in enumerate(rec.log):
        arrays[f"dret{i}"] = _np(r)
    arrays["losses"] = np.array(all_losses, dtype=np.float64)
    meta = dict(kind="reinforce", S=S, A=A, sizes=list(sizes), acts=list(acts), dueling=dueling,
                value_sizes=None if value_sizes is None else list(value_sizes), gamma=gamma,
                lr=lr, wd=wd, off_policy=off_policy, reward_clip=reward_clip,
                clip_param=clip_param, normalize=normalize, subtract_mean=subtract_mean,
                offset_clamp_min=offset_clamp_min, temperature=temperature, seed=seed,
                lengths=list(lengths), n_updates=len(trajs))
    _save(name, arrays, meta)


def ppo_case(name, *, lengths, S=4, A=2, sizes=(32, 32), acts=("leaky_relu", "leaky_relu"),
             dueling=False, value_sizes=None, gamma=0.9, lr=1e-3, wd=0.0, reward_clip=1e6,
             normalize=True, subtract_mean=True, offset_clamp_min=False, update_freq=1,
             update_epochs=1, ppo_batch_size=1, ppo_epsilon=0.2, entropy_weight=0.0,
             td_error_advantage=False, temperature=1.0, masked=False, next_state=False,
             not_terminal=None, constant=(), ratio_noise=0.3, seed=0):
    rlt = ref("reagent.core.types")
    union = ref("reagent.optimizer.union")
    tr = ref("reagent.training.ppo_trainer")
    pol_mod = ref("reagent.gym.policies.policy")
    samp = ref("reagent.gym.policies.samplers.discrete_sampler")
    policy, value = _nets(S, A, sizes, acts, dueling, value_sizes, seed)
    trajs = _trajectories(lengths, S, A, seed + 1, masked=masked, next_state=next_state,
                          not_terminal=not_terminal, constant=constant, policy=policy,
                          temperature=temperature, ratio_noise=ratio_noise)
    assert len(trajs) % update_freq == 0
    trainer = tr.PPOTrainer(
        policy=pol_mod.Policy(scorer=policy, sampler=samp.SoftmaxActionSampler(temperature)),
        gamma=gamma, optimizer=_opt(union, lr, wd), optimizer_value_net=_opt(union, lr, wd),
        actions=[str(i) for i in range(A)], reward_clip=reward_clip, normalize=normalize,
        subtract_mean=subtract_mean, offset_clamp_min=offset_clamp_min, update_freq=update_freq,
        update_epochs=update_epochs, ppo_batch_size=ppo_batch_size, ppo_epsilon=ppo_epsilon,
        entropy_weight=entropy_weight, value_net=value, td_error_advantage=td_error_advantage)
    arrays = {}
    for k, d in enumerate(trajs):
        for f, v in d.items():
            arrays[f"traj{k}.{f}"] = _np(v)
    _dump_net(arrays, "policy0", policy)
    if value is not None:
        _dump_net(arrays, "value0", value)
    # the shims manual optimization needs
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    trainer.optimizers = lambda use_pl_optimizer=True: opts
    trainer.manual_backward = lambda loss, *a, **k: loss.backward()
    trainer.logger = None
    rep = _Reporter(value is not None)
    trainer._reporter = rep
    _grad_recorder(opts, arrays)
    advs = []
    orig_adv = trainer._compute_advantage

    def spy(traj, rewards, ls):
        out = orig_adv(traj, rewards, ls)
        advs.append(out.detach().clone())
        return out

    trainer._compute_advantage = spy
    orig_perm = torch.randperm
    perms = []

    def randperm(n, *a, **k):
        out = orig_perm(n, *a, **k)
        perms.append(out.clone())
        return out

    torch.manual_seed(seed + 2)
    with _Recorder(tr, "discounted_returns") as rec:
        torch.randperm = randperm
        try:
            for k, d in enumerate(trajs):
                trainer.training_step(_rlt_traj(rlt, d), k)
                if (k + 1) % update_freq == 0:
                    u = (k + 1) // update_freq
                    _dump_net(arrays, f"policy{u}", policy)
                    if value is not None:
                        _dump_net(arrays, f"value{u}", value)
        finally:
            torch.randperm = orig_perm
    for i, r in enumerate(rec.log):
        arrays[f"dret{i}"] = _np(r)
    for i, a in enumerate(advs):
        arrays[f"adv{i}"] = _np(a)
    for i, p in enumerate(perms):
        arrays[f"perm{i // update_epochs}.{i % update_epochs}"] = _np(p)
    arrays["losses"] = np.array(rep.losses, dtype=np.float64)
    meta = dict(kind="ppo", S=S, A=A, sizes=list(sizes), acts=list(acts), dueling=dueling,
                value_sizes=None if value_sizes is None else list(value_sizes), gamma=gamma,
                lr=lr, wd=wd, reward_clip=reward_clip, normalize=normalize,
                subtract_mean=subtract_mean, offset_clamp_min=offset_clamp_min,
                update_freq=update_freq, update_epochs=update_epochs,
                ppo_batch_size=ppo_batch_size, ppo_epsilon=ppo_epsilon,
                entropy_weight=entropy_weight, td_error_advantage=td_error_advantage,
                temperature=temperature, seed=seed, lengths=list(lengths),
                n_updates=len(trajs) // update_freq, rng_seed=seed + 2)
    _save(name, arrays, meta)


CASES = [
    # discrete_reinforce_cartpole_online.yaml: gamma 0.99, Adam(1e-3), normalize False,
    # subtract_mean True, FullyConnected [64] leaky_relu, temperature 1
    ("pg_reinforce_cartpole", reinforce_case,
     dict(lengths=[23, 57, 200], gamma=0.99, normalize=False, subtract_mean=True, seed=0)),
    ("pg_reinforce_whiten_offpolicy", reinforce_case,
     dict(lengths=[13, 1, 9], S=7, A=5, sizes=(12, 10), acts=("relu", "tanh"), gamma=0.9,
          off_policy=True, clip_param=1.5, reward_clip=0.5, temperature=0.7, masked=True,
          lr=3e-3, seed=2)),
    ("pg_reinforce_baseline", reinforce_case,
     dict(lengths=[17, 30], S=5, A=3, sizes=(16,), acts=("relu",), value_sizes=(12,),
          gamma=0.95, normalize=False, subtract_mean=False, offset_clamp_min=True, lr=3e-3,
          seed=4)),
    ("pg_reinforce_gamma0_constant", reinforce_case,
     dict(lengths=[6, 11], S=3, A=4, sizes=(8,), acts=("relu",), constant=(0,), lr=3e-3,
          seed=6)),
    # discrete_ppo_cartpole_online.yaml: gamma 0.99, ppo_epsilon 0.2, Adam(1e-3, weight_decay
    # 1e-3), update_freq 2, update_epochs 1, ppo_batch_size 2, FullyConnected [32, 32]
    # leaky_relu, temperature 1
    ("pg_ppo_cartpole", ppo_case,
     dict(lengths=[31, 18, 44, 12, 60, 25], gamma=0.99, wd=1e-3, update_freq=2,
          ppo_batch_size=2, seed=8)),
    ("pg_ppo_baseline_entropy_dueling", ppo_case,
     dict(lengths=[9, 1, 14, 6, 11], S=6, A=3, sizes=(16, 8), acts=("relu", "relu"),
          dueling=True, value_sizes=(10,), gamma=0.9, normalize=False, entropy_weight=0.05,
          update_freq=5, update_epochs=2, ppo_batch_size=3, ratio_noise=0.6, masked=True,
          lr=3e-3, seed=10)),
    ("pg_ppo_td_next_state", ppo_case,
     dict(lengths=[8, 13, 5, 10], S=5, A=3, sizes=(12,), acts=("relu",), value_sizes=(8,),
          gamma=0.95, normalize=False, td_error_advantage=True, next_state=True,
          not_terminal=[1.0, 0.0, 1.0, 0.0], offset_clamp_min=True, update_freq=2,
          ppo_batch_size=2, lr=3e-3, seed=12)),
    ("pg_ppo_td_no_next_state", ppo_case,
     dict(lengths=[7, 12, 3], S=5, A=3, sizes=(12,), acts=("tanh",), value_sizes=(8,),
          gamma=0.9, normalize=False, td_error_advantage=True, update_freq=3,
          ppo_batch_size=2, reward_clip=1.0, temperature=1.3, lr=3e-3, seed=14)),
    ("pg_ppo_whiten_constant", ppo_case,
     dict(lengths=[5, 1, 8], S=3, A=2, sizes=(8,), acts=("relu",), gamma=0.0,
          constant=(0,), update_freq=3, ppo_batch_size=3, seed=16)),
]


def main(only=None):
    for name, fn, kw in CASES:
        if only and name not in only:
            continue
        fn(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
