"""Golden vectors for SlateQ, written to tests/golden/.  Like make_golden.py this runs the
UNMODIFIED reference through oracle/ref_harness.py.

    python oracle/make_slateq_golden.py            # regenerate every case
    python oracle/make_slateq_golden.py NAME ...   # only the named cases

  slateq_recsim_*         five updates of the reference SlateQTrainer wired as the SlateQ
                          manager wires it (model_managers/ranking/slate_q.py: a ParametricDQN
                          FullyConnected critic over (state, item), target = copy) at each RecSim
                          configuration (gym/tests/configs/recsim/slate_q_recsim_online*.yaml),
                          on SlateQInputMaker-shaped batches of 32 rows: slate 3 plus the null slot
                          (index 3), 10 candidates of value augmentation_value and mask 1.  The max-Q
                          configuration gets slate_opt_parameters=TOP_K, without which the
                          reference fails.
  slateq_topk_multi       TOP_K with single_selection=False
  slateq_time_diff        SARSA with a time_diff and discount_time_scale
  slateq_odd_shapes       odd widths, partial candidate masks, random reward masks
  inputmaker_slateq       the reference ReplayBuffer on a seeded RecSim-shaped stream,
                          sample_transition_batch, then SlateQInputMaker
  slateq_scorer           slate_q_scorer and TopKSampler
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


def make_batch(B, C, slate, S, D, gen, *, partial_masks=False, null_slot=True, p_term=0.1,
               time_diff=False):
    """A SlateQInputMaker-shaped batch as plain tensors: each row's slate is `slate` distinct
    candidates, then (null_slot) index `slate`; reward_mask is the clicks plus True on the
    null slot when nothing was clicked (else random)."""
    def slates():
        return torch.stack([torch.randperm(C, generator=gen)[:slate] for _ in range(B)])

    def masks():
        if not partial_masks:
            return torch.ones(B, C)
        m = (torch.rand(B, C, generator=gen) > 0.3).float()
        m[0] = 0.0
        m[0, 0] = 1.0  # row 0: one candidate present
        return m

    act, nact = slates(), slates()
    click = torch.rand(B, slate, generator=gen) < 0.3
    watch = torch.rand(B, slate, generator=gen) * 5 * click
    if null_slot:
        null = torch.full((B, 1), slate, dtype=torch.int64)
        act, nact = torch.cat([act, null], 1), torch.cat([nact, null], 1)
        watch = torch.cat([watch, torch.zeros(B, 1)], 1)
        click = torch.cat([click, (click.sum(1) == 0).view(B, 1)], 1)
    b = dict(state=torch.randn(B, S, generator=gen), docs=torch.randn(B, C, D, generator=gen),
             mask=masks(), value=torch.randn(B, C, generator=gen),
             next_state=torch.randn(B, S, generator=gen),
             next_docs=torch.randn(B, C, D, generator=gen), next_mask=masks(),
             next_value=torch.randn(B, C, generator=gen), action=act, next_action=nact,
             reward=watch, reward_mask=click,
             not_terminal=torch.rand(B, 1, generator=gen) >= p_term)
    if time_diff:
        b["time_diff"] = torch.randint(1, 4, (B, 1), generator=gen).float()
    # float16-representable values, stored as float16 (half the golden's size, exact)
    return {k: v.half().float() if torch.is_floating_point(v) else v for k, v in b.items()}


def _stored(v):
    a = _np(v).copy()
    return a.astype(np.float16) if a.dtype == np.float32 else a


def ref_batch(rlt, b):
    def fd(s, d, m, v):
        return rlt.FeatureData(float_features=s, candidate_docs=rlt.DocList(d, m, v))

    return rlt.SlateQInput(
        state=fd(b["state"], b["docs"], b["mask"], b["value"]),
        next_state=fd(b["next_state"], b["next_docs"], b["next_mask"], b["next_value"]),
        reward=b["reward"], time_diff=b.get("time_diff"), step=None,
        not_terminal=b["not_terminal"], action=b["action"], next_action=b["next_action"],
        reward_mask=b["reward_mask"])


def trainer_case(name, *, B=32, C=10, slate=3, S=20, D=20, sizes=(64, 64),
                 acts=("leaky_relu", "leaky_relu"), gamma=0.9, tau=0.001, lr=1e-3, maxq=False,
                 single_selection=True, norm="norm_by_current_slate_size", time_scale=None,
                 time_diff=False, partial_masks=False, p_term=0.1, seed=0):
    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    critic = ref("reagent.models.critic")
    tr = ref("reagent.training.slate_q_trainer")
    union = ref("reagent.optimizer.union")
    torch.manual_seed(seed)
    q = critic.FullyConnectedCritic(S, D, list(sizes), list(acts))
    with torch.no_grad():  # biases are 0 at init in the reference: exercise the bias paths
        for seq in q.fc.dnn:
            seq[0].bias.normal_(0, 0.1)
    qt = q.get_target_network()
    trainer = tr.SlateQTrainer(
        q, qt, slate, rl=params.RLParameters(gamma=gamma, target_update_rate=tau, maxq_learning=maxq),
        optimizer=union.Optimizer__Union(Adam=union.classes["Adam"](lr=lr)),
        slate_opt_parameters=(params.SlateOptParameters(method=params.SlateOptMethod.TOP_K)
                              if maxq else None),
        discount_time_scale=time_scale, single_selection=single_selection,
        next_slate_value_norm_method=tr.NextSlateValueNormMethod(norm), minibatch_size=B,
        evaluation=params.EvaluationParameters(calc_cpe_in_training=False))
    arrays = {}
    _dump_net(arrays, "q0", q)
    _dump_net(arrays, "qt0", qt)
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    assert type(opts[0]) is torch.optim.Adam, [type(o) for o in opts]
    gen = torch.Generator().manual_seed(seed + 1)
    losses = []
    for it in range(N_UPDATES):
        b = make_batch(B, C, slate, S, D, gen, partial_masks=partial_masks, p_term=p_term,
                       time_diff=time_diff)
        arrays.update({f"batch{it}.{k}": _stored(v) for k, v in b.items()})
        rb = ref_batch(rlt, b)
        out = run_update(trainer, rb, it, opts)
        losses.append(out[0])
        # SARSA: _action_docs zeroed the terminal rows of the batch's next_action in place
        arrays[f"batch{it}.next_action_after"] = _np(rb.next_action).copy()
    arrays["losses"] = np.array(losses, dtype=np.float64)
    _dump_net(arrays, "qN", q)
    _dump_net(arrays, "qtN", qt)
    _save(name, arrays, dict(kind="slateq", B=B, C=C, slate_size=slate, S=S, D=D,
                             sizes=list(sizes), acts=list(acts), gamma=gamma, tau=tau, lr=lr,
                             maxq=maxq, single_selection=single_selection, norm=norm,
                             time_scale=time_scale, time_diff=time_diff,
                             partial_masks=partial_masks, n_updates=N_UPDATES))


def inputmaker_case(name, *, cap=128, n_add=150, B=48, C=10, slate=3, S=20, D=20, seed=30,
                    p_term=0.1, n_samples=2):
    crb = ref("reagent.replay_memory.circular_replay_buffer")
    tp = ref("reagent.gym.preprocessors.trainer_preprocessor")
    rng = np.random.RandomState(seed)
    click = rng.rand(n_add, slate) < 0.3
    st = dict(observation=rng.randn(n_add, S).astype(np.float32),
              action=np.stack([rng.permutation(C)[:slate] for _ in range(n_add)]).astype(np.int64),
              reward=rng.randn(n_add).astype(np.float32),
              terminal=rng.rand(n_add) < p_term,
              doc=rng.randn(n_add, C, D).astype(np.float32),
              augmentation_value=rng.rand(n_add, C).astype(np.float32),
              response_click=click.astype(np.int64),
              response_watch_time=(rng.rand(n_add, slate) * 4 * click).astype(np.float32))
    keys = list(st)
    rb = crb.ReplayBuffer(stack_size=1, replay_capacity=cap, batch_size=B)
    for t in range(n_add):
        kw = {}
        for k in keys:
            v = st[k][t]
            if k == "terminal":
                v = bool(v)
            elif np.ndim(v) == 0:
                v = float(v)
            kw[k] = v
        rb.add(**kw)
    arrays = {f"stream.{k}": st[k] for k in keys}
    maker = tp.SlateQInputMaker()
    random.seed(seed + 200)
    np.random.seed(seed + 200)
    torch.manual_seed(seed + 200)
    for s_i in range(n_samples):
        raw = rb.sample_transition_batch(batch_size=B)
        out = maker(raw)
        pre = f"sample{s_i}."
        arrays[pre + "indices"] = _np(raw.indices)
        got = dict(state=out.state.float_features, next_state=out.next_state.float_features,
                   docs=out.state.candidate_docs.float_features,
                   next_docs=out.next_state.candidate_docs.float_features,
                   mask=out.state.candidate_docs.mask, next_mask=out.next_state.candidate_docs.mask,
                   value=out.state.candidate_docs.value,
                   next_value=out.next_state.candidate_docs.value, action=out.action,
                   next_action=out.next_action, reward=out.reward, reward_mask=out.reward_mask,
                   not_terminal=out.not_terminal)
        assert out.time_diff is None
        for k, v in got.items():
            arrays[pre + k] = _np(v)
    _save(name, arrays, dict(kind="inputmaker_slateq", cap=cap, n_add=n_add, B=B, C=C,
                             slate_size=slate, S=S, D=D, seed=seed, n_samples=n_samples,
                             keys=keys))


def scorer_case(name, *, n=37, C=10, slate=3, S=20, D=20, sizes=(64, 64),
                acts=("leaky_relu", "leaky_relu"), seed=40):
    rlt = ref("reagent.core.types")
    critic = ref("reagent.models.critic")
    sc = ref("reagent.gym.policies.scorers.slate_q_scorer")
    ts = ref("reagent.gym.policies.samplers.top_k_sampler")
    torch.manual_seed(seed)
    q = critic.FullyConnectedCritic(S, D, list(sizes), list(acts))
    with torch.no_grad():
        for seq in q.fc.dnn:
            seq[0].bias.normal_(0, 0.1)
    gen = torch.Generator().manual_seed(seed + 1)
    obs = torch.randn(n, S, generator=gen)
    docs = torch.randn(n, C, D, generator=gen)
    value = torch.rand(n, C, generator=gen)
    arrays = {"obs": _np(obs), "docs": _np(docs), "value": _np(value)}
    _dump_net(arrays, "q", q)
    state = rlt.FeatureData(float_features=obs, candidate_docs=rlt.DocList(docs, value=value))
    scores = sc.slate_q_scorer(num_candidates=C, q_network=q)(state)
    assert q.training
    arrays["scores"] = _np(scores)
    out = ts.TopKSampler(k=slate).sample_action(scores)
    arrays["action"] = _np(out.action)
    arrays["log_prob"] = _np(out.log_prob)
    _save(name, arrays, dict(kind="slateq_scorer", n=n, C=C, slate_size=slate, S=S, D=D,
                             sizes=list(sizes), acts=list(acts), seed=seed))


def main(only=None):
    cases = []

    def add(fn, name, **kw):
        cases.append((fn, name, kw))

    # gym/tests/configs/recsim/*.yaml: slate 3, 10 candidates, [64, 64] leaky_relu, Adam 1e-3
    add(trainer_case, "slateq_recsim_online", seed=1)
    add(trainer_case, "slateq_recsim_online_with_time_scale", time_scale=2.0, seed=2)
    add(trainer_case, "slateq_recsim_online_multi_selection", single_selection=False,
        norm="norm_by_next_slate_size", seed=3)
    add(trainer_case, "slateq_recsim_online_multi_selection_avg_curr", single_selection=False,
        norm="norm_by_current_slate_size", seed=4)
    add(trainer_case, "slateq_recsim_online_maxq_topk", maxq=True, seed=5)
    add(trainer_case, "slateq_topk_multi", maxq=True, single_selection=False,
        norm="norm_by_next_slate_size", seed=6)
    add(trainer_case, "slateq_time_diff", time_scale=2.0, time_diff=True, gamma=0.95, tau=0.1,
        seed=7)
    add(trainer_case, "slateq_odd_shapes", B=37, C=7, slate=2, S=5, D=3, sizes=(24, 12),
        acts=("relu", "tanh"), partial_masks=True, p_term=0.25, gamma=0.8, tau=0.2, lr=1e-2,
        seed=8)
    add(inputmaker_case, "inputmaker_slateq")
    add(scorer_case, "slateq_scorer")
    for fn, name, kw in cases:
        if only and name not in only:
            continue
        fn(name, **kw)


if __name__ == "__main__":
    main(sys.argv[1:] or None)
