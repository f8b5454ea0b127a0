"""REINFORCE and PPO on the GPU: rb200_pg_returns bit for bit against the reference's
discounted_returns, both trainers against every golden of the unmodified reference (REINFORCE
through the generator and train_batch, which agree bit for bit; PPO through training_step /
update_model with the reference's permutations), the manager-built PPO CartPole
configuration, and the grow-only workspace."""
import numpy as np
import pytest
import torch

from oracle import pg_oracle as PO
from tests import golden_util as G
from tests import pg_cases as P

pytestmark = pytest.mark.gpu


def _returns(rewards, lengths, *, gamma, reward_clip=1e6, norm=0, clamp_min=False):
    from reagent_b200 import _lib

    dev = torch.device("cuda")
    r = torch.cat([x.reshape(-1) for x in rewards]).float().to(dev).contiguous()
    offs = torch.tensor(PO.pack_offsets(lengths), dtype=torch.int32, device=dev)
    out = torch.full_like(r, float("nan"))
    a = _lib.PgReturnsArgsT()
    a.n_traj, a.offsets, a.reward = len(lengths), offs.data_ptr(), r.data_ptr()
    a.reward_clip, a.gamma, a.norm, a.offset_clamp_min = reward_clip, gamma, norm, int(clamp_min)
    a.returns = out.data_ptr()
    _lib.check(_lib.lib().rb200_pg_returns(a, _lib.cur_stream()), "rb200_pg_returns")
    return out.cpu()


def test_returns_bit_identical_to_the_fp32_loop_at_every_length():
    g = torch.Generator().manual_seed(0)
    lengths = [1, 7, 200, 10000, 129, 128]
    rewards = [torch.randn(n, generator=g) * 3 for n in lengths]
    for gamma in (0.99, 0.5, 0.0):
        got = _returns(rewards, lengths, gamma=gamma, reward_clip=2.5)
        want = torch.cat([PO.discounted_returns(torch.clamp(r, max=2.5), gamma) for r in rewards])
        assert torch.equal(got, want), gamma


@pytest.mark.parametrize("name", P.REINFORCE_CASES)
def test_returns_bit_identical_to_reference_discounted_returns(name):
    arrays, meta = G.load(name)
    trajs = P.trajectories(arrays)
    rewards = [t["reward"] for t in trajs]
    got = _returns(rewards, [len(r) for r in rewards], gamma=meta["gamma"],
                   reward_clip=meta["reward_clip"])
    want = np.concatenate([arrays[f"dret{k}"] for k in range(len(trajs))])
    assert np.array_equal(got.numpy(), want)


@pytest.mark.parametrize("norm,subtract,gamma", [(1, True, 0.0), (1, True, 0.9), (2, False, 0.9),
                                                 (3, True, 0.0)])
def test_normalized_returns_match_fp64(norm, subtract, gamma):
    g = torch.Generator().manual_seed(1)
    lengths = [1, 6, 33, 500]
    rewards = [torch.randn(n, generator=g) for n in lengths]
    rewards[1] = torch.ones(6)  # constant: whitening gives 0 when gamma is 0
    got = _returns(rewards, lengths, gamma=gamma, norm=norm, clamp_min=True)
    want = PO.returns_fp64(torch.cat(rewards), PO.pack_offsets(lengths), gamma=gamma,
                           reward_clip=1e6, normalize=norm in (1, 2), subtract_mean=subtract,
                           offset_clamp_min=True)
    assert G.rel_err(got, want) < 1e-5
    if subtract:  # a length-1 trajectory is its own mean
        assert float(got[0]) == 0.0
    if norm == 1 and gamma == 0.0:
        assert torch.equal(got[1:7], torch.zeros(6))


def _build(meta, arrays, kind):
    from reagent_b200.gym.policies import Policy, SoftmaxActionSampler
    from reagent_b200.models import DuelingQNetwork, FullyConnectedDQN
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import PPOTrainer, ReinforceTrainer

    S, A = meta["S"], meta["A"]
    if meta["dueling"]:
        net = DuelingQNetwork.make_fully_connected(S, A, meta["sizes"], meta["acts"])
    else:
        net = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"])
    G.load_into_module(arrays, "policy0", net)
    value = None
    if meta["value_sizes"] is not None:
        value = FloatFeatureFullyConnected(S, 1, meta["value_sizes"],
                                           ["relu"] * len(meta["value_sizes"]))
        G.load_into_module(arrays, "value0", value)
        value = value.cuda()
    net = net.cuda()
    opt = lambda: Optimizer__Union.default(lr=meta["lr"], weight_decay=meta["wd"])  # noqa: E731
    pol = Policy(scorer=net, sampler=SoftmaxActionSampler(meta["temperature"]))
    if kind == "reinforce":
        kw = {k: meta[k] for k in ("gamma", "off_policy", "reward_clip", "clip_param",
                                   "normalize", "subtract_mean", "offset_clamp_min")}
        return ReinforceTrainer(pol, optimizer=opt(), optimizer_value_net=opt(), value_net=value,
                                **kw).cuda()
    kw = {k: meta[k] for k in ("gamma", "reward_clip", "normalize", "subtract_mean",
                               "offset_clamp_min", "update_freq", "update_epochs",
                               "ppo_batch_size", "ppo_epsilon", "entropy_weight",
                               "td_error_advantage")}
    return PPOTrainer(pol, optimizer=opt(), optimizer_value_net=opt(), value_net=value,
                      **kw).cuda()


def _params(net):
    return [p.detach().cpu() for p in net.parameters()]


@pytest.mark.parametrize("name", P.REINFORCE_CASES)
def test_reinforce_matches_reference_generator_and_train_batch(name):
    from reagent_b200.training import run_update

    arrays, meta = G.load(name)
    slow, fast = _build(meta, arrays, "reinforce"), _build(meta, arrays, "reinforce")
    for u, t in enumerate(P.trajectories(arrays, "cuda")):
        batch = P.as_input(t)
        losses = [float(l) for l in run_update(slow, batch, u)]
        P.check_losses(losses, arrays["losses"][u])
        # the advantage against the oracle from the reference's parameters before this update
        pol_u, val_u = P.oracle_nets(arrays, meta, u)
        want_adv = PO.reinforce_update(pol_u, val_u, P.adam(meta, pol_u), P.adam(meta, val_u),
                                       {k: v.cpu() for k, v in t.items()},
                                       **P.reinforce_kwargs(meta))[3]
        assert G.rel_err(slow.advantage(len(t["reward"])), want_adv) < G.TOL
        ret = slow.returns(len(t["reward"])).cpu()
        if not meta["normalize"] and not meta["subtract_mean"] and not meta["offset_clamp_min"]:
            assert np.array_equal(ret.numpy(), arrays[f"dret{u}"])
        if u == 0:
            nets = ([slow.value_net] if slow.value_net is not None else []) + [slow.scorer]
            for oi, net in enumerate(nets):
                P.check_grads(arrays, oi, [g.cpu() for g in slow.net_grads(net)])
        fl = fast.train_batch(batch, u)
        got = [float(fl[1])] if fast.value_net is not None else []
        assert got + [float(fl[0])] == losses
        P.check_net(arrays, f"policy{u + 1}", _params(slow.scorer))
        for a, b in zip(_params(slow.scorer), _params(fast.scorer)):
            assert torch.equal(a, b)
        if slow.value_net is not None:
            P.check_net(arrays, f"value{u + 1}", _params(slow.value_net))
            for a, b in zip(_params(slow.value_net), _params(fast.value_net)):
                assert torch.equal(a, b)


class _Reporter:
    def __init__(self):
        self.logged = []

    def log(self, **kw):
        self.logged.append({k: float(v) for k, v in kw.items()})


def _run_ppo(trainer, arrays, meta, trajs):
    rep = _Reporter()
    trainer.set_reporter(rep)
    perms = []
    orig = torch.randperm

    def randperm(n, *a, **k):
        out = orig(n, *a, **k)
        perms.append(out.clone())
        return out

    torch.manual_seed(meta["rng_seed"])
    torch.randperm = randperm
    try:
        for k, t in enumerate(trajs):
            trainer.training_step(P.as_input(t), k)
            if (k + 1) % meta["update_freq"] == 0:
                u = (k + 1) // meta["update_freq"]
                ps = _params(trainer.scorer)
                P.check_net(arrays, f"policy{u}", ps, skip=P.value_head_free(meta, len(ps)))
                if trainer.value_net is not None:
                    P.check_net(arrays, f"value{u}", _params(trainer.value_net))
    finally:
        torch.randperm = orig
    for i, p in enumerate(perms):
        assert np.array_equal(p.numpy(), arrays[f"perm{i // meta['update_epochs']}."
                                               f"{i % meta['update_epochs']}"])
    for m, row in enumerate(arrays["losses"]):
        got = ([rep.logged[m]["value_net_loss"]] if trainer.value_net is not None else [])
        P.check_losses(got + [rep.logged[m]["ppo_loss"]], row)
    assert len(rep.logged) == len(arrays["losses"])


@pytest.mark.parametrize("name", P.PPO_CASES)
def test_ppo_matches_reference(name):
    arrays, meta = G.load(name)
    trajs = P.trajectories(arrays, "cuda")
    # the first minibatch alone: advantages and gradients
    t = _build(meta, arrays, "ppo")
    _, idx = P.minibatches(arrays, meta)[0]
    t._losses([P.as_input(trajs[i]) for i in idx])
    rows = sum(len(trajs[i]["reward"]) for i in idx)
    want = np.concatenate([arrays[f"adv{j}"] for j in range(len(idx))])
    assert G.rel_err(t.advantage(rows), want) < G.TOL
    nets = ([t.value_net] if t.value_net is not None else []) + [t.scorer]
    for oi, net in enumerate(nets):
        P.check_grads(arrays, oi, [g.cpu() for g in t.net_grads(net)])
    _run_ppo(_build(meta, arrays, "ppo"), arrays, meta, trajs)


def test_ppo_cartpole_through_the_manager():
    from reagent_b200 import model_managers as M
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters
    from reagent_b200.net_builder import FullyConnected
    from reagent_b200.optimizer import Optimizer__Union

    arrays, meta = G.load("pg_ppo_cartpole")
    m = M.PPO(actions=["0", "1"], gamma=0.99, ppo_epsilon=0.2,
              optimizer=Optimizer__Union.default(lr=0.001, weight_decay=0.001), update_freq=2,
              update_epochs=1, ppo_batch_size=2,
              policy_net_builder=FullyConnected(sizes=[32, 32],
                                                activations=["leaky_relu", "leaky_relu"]))
    nd = NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS") for i in range(4)})
    trainer = m.build_trainer({"state": nd}, use_gpu=True)
    assert trainer.scorer.arena.dims == [4, 32, 32, 2]
    assert m.create_policy(trainer).scorer is trainer.scorer
    assert m.create_policy(trainer) is m._create_policy(None)
    with torch.no_grad():
        G.load_into_module(arrays, "policy0", trainer.scorer)
    _run_ppo(trainer, arrays, meta, P.trajectories(arrays, "cuda"))


def test_workspace_grows_only():
    from reagent_b200.core import types as rlt
    from reagent_b200.gym.policies import Policy, SoftmaxActionSampler
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import ReinforceTrainer

    torch.manual_seed(0)
    t = ReinforceTrainer(Policy(scorer=FullyConnectedDQN(4, 2, [64], ["leaky_relu"]).cuda(),
                                sampler=SoftmaxActionSampler()), gamma=0.99).cuda()

    def traj(n):
        return rlt.PolicyGradientInput(
            state=rlt.FeatureData(torch.randn(n, 4, device="cuda")),
            action=torch.eye(2, device="cuda")[torch.randint(2, (n,), device="cuda")],
            reward=torch.ones(n, device="cuda"), log_prob=torch.zeros(n, device="cuda"))

    for n in (5, 300, 17):
        t.train_batch(traj(n))
    ws = t._pg.ws
    ptrs = {k: v.data_ptr() for k, v in ws.items() if isinstance(v, torch.Tensor)}
    slabs = {k: v.data_ptr() for k, v in t._pg._slabs.items()}
    for n in (1, 299, 300, 64, 2, 150):
        t.train_batch(traj(n))
        assert t._pg.ws is ws and ws["rows"] == 300
        assert {k: v.data_ptr() for k, v in ws.items() if isinstance(v, torch.Tensor)} == ptrs
        assert {k: v.data_ptr() for k, v in t._pg._slabs.items()} == slabs
    torch.cuda.synchronize()
    assert all(torch.isfinite(p).all() for p in t.scorer.parameters())


def test_updates_do_not_synchronise():
    """REINFORCE's train_batch (with a value baseline) and PPO's _update_model (whitening, a
    minibatch in which only some trajectories carry next_state, which only the TD advantage
    reads) launch without waiting on the GPU: packing copies its offsets from pinned memory."""
    from reagent_b200.core import types as rlt
    from reagent_b200.gym.policies import Policy, SoftmaxActionSampler
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.training import PPOTrainer, ReinforceTrainer

    torch.manual_seed(0)

    def policy():
        return Policy(scorer=FullyConnectedDQN(4, 3, [16], ["relu"]).cuda(),
                      sampler=SoftmaxActionSampler())

    def traj(n, next_state=False):
        return rlt.PolicyGradientInput(
            state=rlt.FeatureData(torch.randn(n, 4, device="cuda")),
            action=torch.eye(3, device="cuda")[torch.randint(3, (n,), device="cuda")],
            reward=torch.randn(n, device="cuda"), log_prob=-torch.rand(n, device="cuda"),
            next_state=rlt.FeatureData(torch.randn(n, 4, device="cuda")) if next_state else None)

    value = FloatFeatureFullyConnected(4, 1, [8], ["relu"]).cuda()
    rt = ReinforceTrainer(policy(), gamma=0.9, value_net=value, normalize=False,
                          subtract_mean=False).cuda()
    pt = PPOTrainer(policy(), gamma=0.9, update_freq=3, ppo_batch_size=3).cuda()
    batches = [traj(30), traj(12)]
    mini = [traj(9), traj(14, next_state=True), traj(5)]
    rt.train_batch(batches[0])  # first calls: optimizer state, workspaces
    pt._update_model(mini)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b in batches:
            rt.train_batch(b)
        pt._update_model(mini)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(rt._pg.ws["loss"]).all() and torch.isfinite(pt.last_losses).all()
