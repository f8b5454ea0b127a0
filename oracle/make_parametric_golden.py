"""Golden vectors for ParametricDQN end to end, written to tests/golden/.  Like make_golden.py this
runs the UNMODIFIED reference through oracle/ref_harness.py.

    python oracle/make_parametric_golden.py            # regenerate every case
    python oracle/make_parametric_golden.py NAME ...   # only the named cases

  inputmaker_parametric_*   the reference ReplayBuffer / PrioritizedReplayBuffer on a seeded
                            transition stream, sample_transition_batch, then
                            ParametricDqnInputMaker (gym/preprocessors/trainer_preprocessor.py:370-413)
  pdqn_*_cartpole           five updates of the reference ParametricDQNTrainer wired as the
                            ParametricDQN manager wires it (model_managers/parametric/
                            parametric_dqn.py:45-81: q network, reward network with one output,
                            target = copy of q) at the two CartPole configurations
                            (gym/tests/configs/cartpole/parametric_{dqn,sarsa}_cartpole_online.yaml),
                            each update on its own seeded ParametricDqnInputMaker-shaped batch
  parametric_scorer         parametric_dqn_scorer (gym/policies/scorers/discrete_scorer.py:65-87)
                            and SoftmaxActionSampler draws after torch.manual_seed
"""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle.make_golden import _dump_net, _np, _save  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402

N_UPDATES = 5


# ---------------------------------------------------------------------------
# ParametricDqnInputMaker on a sampled reference batch
# ---------------------------------------------------------------------------
def inputmaker_case(name, *, prioritized, cap, n_add, B, A, horizon=1, gamma=0.9, S=6, seed=0,
                    p_term=0.08, with_masks=False, n_samples=2):
    crb = ref("reagent.replay_memory.circular_replay_buffer")
    prb = ref("reagent.replay_memory.prioritized_replay_buffer")
    tp = ref("reagent.gym.preprocessors.trainer_preprocessor")
    rng = np.random.RandomState(seed)
    st = dict(observation=rng.randn(n_add, S).astype(np.float32),
              action=rng.randint(0, A, size=n_add).astype(np.int64),
              reward=rng.randn(n_add).astype(np.float32),
              terminal=(rng.rand(n_add) < p_term),
              log_prob=(-rng.rand(n_add) * 2).astype(np.float32),
              priority=rng.uniform(0.1, 10.0, size=n_add))
    keys = ["observation", "action", "reward", "terminal", "log_prob"]
    if with_masks:  # stored, and ignored by ParametricDqnInputMaker
        st["possible_actions_mask"] = (rng.rand(n_add, A) > 0.5).astype(np.float32)
        keys.append("possible_actions_mask")
    if prioritized:
        keys.append("priority")
    cls = prb.PrioritizedReplayBuffer if prioritized else crb.ReplayBuffer
    rb = cls(stack_size=1, replay_capacity=cap, batch_size=B, update_horizon=horizon, gamma=gamma)
    for t in range(n_add):
        kw = {}
        for k in keys:
            v = st[k][t]
            if k == "terminal":
                v = bool(v)
            elif k == "priority":
                v = float(v)
            elif k == "action":
                v = int(v)
            elif np.ndim(v) == 0:
                v = float(v)
            kw[k] = v
        rb.add(**kw)
    arrays = {f"stream.{k}": st[k] for k in keys}
    maker = tp.ParametricDqnInputMaker(num_actions=A)
    random.seed(seed + 200)
    torch.manual_seed(seed + 200)
    np.random.seed(seed + 200)
    for s_i in range(n_samples):
        raw = rb.sample_transition_batch(batch_size=B)
        out = maker(raw)
        pre = f"sample{s_i}."
        arrays[pre + "indices"] = _np(raw.indices)
        arrays[pre + "terminal"] = _np(raw.terminal)
        assert out.step is None and out.time_diff is None
        got = dict(state=out.state.float_features, next_state=out.next_state.float_features,
                   action=out.action.float_features, next_action=out.next_action.float_features,
                   possible_actions=out.possible_actions.float_features,
                   possible_next_actions=out.possible_next_actions.float_features,
                   possible_actions_mask=out.possible_actions_mask,
                   possible_next_actions_mask=out.possible_next_actions_mask,
                   reward=out.reward, not_terminal=out.not_terminal,
                   action_probability=out.extras.action_probability)
        for k, v in got.items():
            arrays[pre + k] = _np(v)
    meta = dict(kind="inputmaker_parametric", prioritized=prioritized, cap=cap, n_add=n_add, B=B,
                horizon=horizon, gamma=gamma, S=S, A=A, seed=seed, with_masks=with_masks,
                n_samples=n_samples, keys=keys)
    _save(name, arrays, meta)


# ---------------------------------------------------------------------------
# the reference trainer as the ParametricDQN manager builds it, at the CartPole configurations
# ---------------------------------------------------------------------------
def _batch(rlt, B, S, A, gen):
    """A ParametricDqnInputMaker-shaped batch: one-hot actions, the next one zeroed on terminal
    rows, the identity tiling as the possible actions, ones masks."""
    act = torch.randint(A, (B,), generator=gen)
    nact = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.1).float()
    eye = torch.eye(A).repeat(B, 1)
    batch = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
                 reward=torch.randn(B, 1, generator=gen), not_terminal=nt,
                 action=torch.nn.functional.one_hot(act, A).float(),
                 next_action=torch.nn.functional.one_hot(nact, A).float() * nt,
                 possible_actions=eye, possible_next_actions=eye.clone(),
                 possible_actions_mask=torch.ones(B, A),
                 possible_next_actions_mask=torch.ones(B, A))
    rbatch = rlt.ParametricDqnInput(
        state=rlt.FeatureData(batch["state"]), next_state=rlt.FeatureData(batch["next_state"]),
        reward=batch["reward"], time_diff=None, step=None, not_terminal=nt,
        action=rlt.FeatureData(batch["action"]), next_action=rlt.FeatureData(batch["next_action"]),
        possible_actions=rlt.FeatureData(batch["possible_actions"]),
        possible_actions_mask=batch["possible_actions_mask"],
        possible_next_actions=rlt.FeatureData(batch["possible_next_actions"]),
        possible_next_actions_mask=batch["possible_next_actions_mask"], extras=rlt.ExtraData())
    return batch, rbatch


def cartpole_case(name, *, sizes, acts, gamma, tau, maxq, temperature, optimizer, lr,
                  amsgrad=False, weight_decay=0.0, B=1024, S=4, A=2, seed=0):
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    critic = ref("reagent.models.critic")
    tr = ref("reagent.training.parametric_dqn_trainer")
    union = ref("reagent.optimizer.union")
    if optimizer == "AdamW":
        opt = union.Optimizer__Union(AdamW=union.classes["AdamW"](
            lr=lr, weight_decay=weight_decay, amsgrad=amsgrad))
    else:
        opt = union.Optimizer__Union(Adam=union.classes["Adam"](lr=lr))
    torch.manual_seed(seed)
    # net_builder/parametric_dqn/fully_connected.py: FullyConnectedCritic(state_dim, action_dim,
    # sizes, activations, output_dim); the reward network has len(metrics_to_score) + 1 = 1 output
    q = critic.FullyConnectedCritic(S, A, list(sizes), list(acts))
    rn = critic.FullyConnectedCritic(S, A, list(sizes), list(acts), output_dim=1)
    qt = q.get_target_network()
    rl = params.RLParameters(gamma=gamma, target_update_rate=tau, maxq_learning=maxq,
                             temperature=temperature)
    trainer = tr.ParametricDQNTrainer(q, qt, rn, rl=rl, double_q_learning=True,
                                      minibatches_per_step=1, optimizer=opt)
    arrays = {}
    _dump_net(arrays, "q0", q)
    _dump_net(arrays, "qt0", qt)
    _dump_net(arrays, "r0", rn)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    want = torch.optim.AdamW if optimizer == "AdamW" else torch.optim.Adam
    assert type(opts[0]) is want and type(opts[1]) is want, [type(o) for o in opts]
    gen = torch.Generator().manual_seed(seed + 1)
    losses = []
    for it in range(N_UPDATES):
        batch, rbatch = _batch(rlt, B, S, A, gen)
        arrays.update({f"batch{it}.{k}": _np(v) for k, v in batch.items()})
        out = run_update(trainer, rbatch, it, opts)
        losses.append(out[:2])
    arrays["losses"] = np.array(losses, dtype=np.float64)
    _dump_net(arrays, "qN", q)
    _dump_net(arrays, "qtN", qt)
    _dump_net(arrays, "rN", rn)
    _save(name, arrays, dict(kind="pdqn_cartpole", B=B, S=S, A=A, sizes=list(sizes),
                             acts=list(acts), gamma=gamma, tau=tau, maxq=maxq,
                             temperature=temperature, optimizer=optimizer, lr=lr,
                             amsgrad=amsgrad, weight_decay=weight_decay, double_q=True,
                             n_updates=N_UPDATES))


# ---------------------------------------------------------------------------
# parametric_dqn_scorer + SoftmaxActionSampler
# ---------------------------------------------------------------------------
def scorer_case(name, *, n=37, S=4, A=2, sizes=(128, 64), acts=("leaky_relu", "leaky_relu"),
                temperatures=(1.0, 0.35), n_draws=3, seed=0):
    rlt = ref("reagent.core.types")
    critic = ref("reagent.models.critic")
    sc = ref("reagent.gym.policies.scorers.discrete_scorer")
    ds = ref("reagent.gym.policies.samplers.discrete_sampler")
    torch.manual_seed(seed)
    q = critic.FullyConnectedCritic(S, A, list(sizes), list(acts))
    with torch.no_grad():  # biases are 0 at init in the reference: exercise the bias paths
        for seq in q.fc.dnn:
            seq[0].bias.normal_(0, 0.1)
    obs = torch.randn(n, S, generator=torch.Generator().manual_seed(seed + 1)) * 2
    arrays = {"obs": _np(obs)}
    _dump_net(arrays, "q", q)
    scores = sc.parametric_dqn_scorer(max_num_actions=A, q_network=q)(rlt.FeatureData(obs))
    assert q.training
    arrays["scores"] = _np(scores)
    for ti, temp in enumerate(temperatures):
        sm = ds.SoftmaxActionSampler(temperature=temp)
        for d in range(n_draws):
            torch.manual_seed(seed + 100 * (ti + 1) + d)
            out = sm.sample_action(scores)
            arrays[f"t{ti}.d{d}.action"] = _np(out.action)
            arrays[f"t{ti}.d{d}.log_prob"] = _np(out.log_prob)
    _save(name, arrays, dict(kind="parametric_scorer", n=n, S=S, A=A, sizes=list(sizes),
                             acts=list(acts), temperatures=list(temperatures), n_draws=n_draws,
                             seed=seed))


def main(only=None):
    cases = []

    def add(fn, name, **kw):
        cases.append((fn, name, kw))

    add(inputmaker_case, "inputmaker_parametric_uniform_terminal", prioritized=False, cap=256,
        n_add=200, B=48, A=3, seed=10, p_term=0.3)
    add(inputmaker_case, "inputmaker_parametric_h3_wrap", prioritized=False, cap=128, n_add=300,
        B=40, A=4, seed=11, horizon=3, gamma=0.95)
    add(inputmaker_case, "inputmaker_parametric_masks_logprob", prioritized=False, cap=256,
        n_add=180, B=32, A=5, seed=12, with_masks=True)
    add(inputmaker_case, "inputmaker_parametric_per", prioritized=True, cap=256, n_add=230, B=48,
        A=2, seed=13, horizon=2, gamma=0.9)
    add(cartpole_case, "pdqn_adamw_amsgrad_cartpole", sizes=(128, 64),
        acts=("leaky_relu", "leaky_relu"), gamma=0.99, tau=0.1, maxq=True, temperature=1.0,
        optimizer="AdamW", lr=1e-3, amsgrad=True, weight_decay=0.01, seed=20)
    add(cartpole_case, "pdqn_sarsa_adam_cartpole", sizes=(64, 64),
        acts=("leaky_relu", "leaky_relu"), gamma=0.99, tau=0.2, maxq=False, temperature=0.35,
        optimizer="Adam", lr=0.05, seed=21)
    add(scorer_case, "parametric_scorer")
    for fn, name, kw in cases:
        if only and name not in only:
            continue
        fn(name, **kw)


if __name__ == "__main__":
    main(sys.argv[1:] or None)
