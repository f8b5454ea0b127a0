"""Prioritized replay and the captured online step for SACTrainer and TD3Trainer on the GPU:
importance-weighted critics against the weighted oracle, the twin-critic TD errors and
priorities, and FusedPolicyStep(rng="device", online=True, per=...) against a host replica of the
reference buffer, captured against eager, and against train_batch on the same indices."""
import random

import numpy as np
import pytest
import torch

from oracle import per_ac_oracle as PA
from oracle import td_oracle as O
from tests import golden_util as G
from tests.online_step import (assert_captured_equals_eager, assert_matches_host_replica,
                               assert_nan_reward_raises, bench_setup, filled_heap, host_add,
                               rows_update, transition_stream, tree, ulps)
from tests.builders import _build_sac, _build_td3, _inject, _net_arrays, _pbatch, _rand_net
from tests.golden_cases import SAC_CASES, TD3_CASES
from tests.golden_util import _adam_close

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _golden(name):
    """(trainer, gpu batch, oracle state, cpu batch, meta, arrays)"""
    arrays, meta = G.load(name)
    batch = G.batch_tensors(arrays)
    gb = _pbatch(G.batch_tensors(arrays, "cuda"))
    if name.startswith("sac"):
        acts = meta["acts"] + ["linear"]
        st = O.SacState(G.oracle_net(arrays, "actor0", acts), G.oracle_net(arrays, "q1_0", acts),
                        G.oracle_net(arrays, "q2_0", acts) if meta["twin"] else None,
                        lr=meta["lr"], entropy_temperature=meta["entropy_temperature"],
                        learn_alpha=meta["learn_alpha"], target_entropy=meta["target_entropy"])
        return _build_sac(meta, arrays), gb, st, batch, meta, arrays
    cacts = meta["acts"] + ["linear"]
    st = O.Td3State(G.oracle_net(arrays, "actor0", meta["acts"] + ["tanh"]),
                    G.oracle_net(arrays, "q1_0", cacts),
                    G.oracle_net(arrays, "q2_0", cacts) if meta["twin"] else None, lr=meta["lr"])
    return _build_td3(meta, arrays), gb, st, batch, meta, arrays


def _modules(t):
    """Every trained network of the trainer (online and target), in a fixed order."""
    mods = [t.actor_network, t.q1_network, t.q1_network_target]
    if t.q2_network is not None:
        mods += [t.q2_network, t.q2_network_target]
    if hasattr(t, "actor_network_target"):
        mods.append(t.actor_network_target)
    return mods


def _state(t):
    out = [p.detach().clone() for m in _modules(t) for p in m.parameters()]
    if hasattr(t, "log_alpha"):
        out += [t.log_alpha.detach().clone(), t._alpha_dev.clone()]
    return out


def _oracle_modules(t, st):
    pairs = [(t.actor_network, st.actor), (t.q1_network, st.q1), (t.q1_network_target, st.q1t)]
    if t.q2_network is not None:
        pairs += [(t.q2_network, st.q2), (t.q2_network_target, st.q2t)]
    if hasattr(t, "actor_network_target"):
        pairs.append((t.actor_network_target, st.actor_t))
    return pairs


def _cmp_net(mod, net, tol, what):
    for i, seq in enumerate(mod.fc.dnn):
        assert G.rel_err(seq[0].weight, net["W"][i].detach()) < tol, (what, "W", i)
        assert G.rel_err(seq[0].bias, net["b"][i].detach()) < tol, (what, "b", i)


@pytest.mark.parametrize("name", ["sac_twin_alpha", "sac_single_fixed_alpha", "td3_twin",
                                  "td3_single"])
def test_unit_weights_are_bit_identical_to_unweighted(name):
    runs = []
    for weighted in (False, True):
        t, gb, _, _, meta, arrays = _golden(name)
        w = torch.ones(meta["B"], device="cuda") if weighted else None
        losses, rows = [], []
        for it in range(meta["n_updates"]):
            _inject(t, arrays, it)
            closs, aloss = t.train_batch(gb, it, importance_weights=w)
            losses.append(closs.clone())
            if aloss is not None:
                losses.append(aloss.clone())
            rows.append([t._ws[k].clone() for k in ("td_target", "q1_value", "q2_value")]
                        if meta["twin"] else [t._ws[k].clone() for k in ("td_target", "q1_value")])
        runs.append((losses, rows, _state(t)))
    (l0, r0, s0), (l1, r1, s1) = runs
    assert len(l0) == len(l1) and all(torch.equal(a, b) for a, b in zip(l0, l1))
    assert all(torch.equal(a, b) for x, y in zip(r0, r1) for a, b in zip(x, y))
    assert all(torch.equal(a, b) for a, b in zip(s0, s1))


@pytest.mark.parametrize("name", SAC_CASES + TD3_CASES)
def test_weighted_update_matches_oracle(name):
    """Random weights in [0.05, 1] on the golden batches, the reference's noise injected: critic
    losses, td_target, q values and TD errors of every update, and every post-update network."""
    t, gb, st, batch, meta, arrays = _golden(name)
    sac = name.startswith("sac")
    gen = torch.Generator().manual_seed(1)
    for it in range(meta["n_updates"]):
        w = 0.05 + 0.95 * torch.rand(meta["B"], generator=gen)
        nn_ = torch.from_numpy(arrays[f"noise{it}.next"])
        _inject(t, arrays, it)
        closs, _ = t.train_batch(gb, it, importance_weights=w.cuda())
        if sac:
            out = PA.weighted_sac_update(st, batch, nn_, torch.from_numpy(arrays[f"noise{it}.cur"]),
                                         w, gamma=meta["gamma"], tau=meta["tau"],
                                         backprop_through_log_prob=meta["backprop"])
        else:
            out = PA.weighted_td3_update(st, batch, nn_, it, w, gamma=meta["gamma"], tau=meta["tau"],
                                         noise_variance=meta["noise_variance"],
                                         noise_clip=meta["noise_clip"],
                                         delayed_policy_update=meta["delay"])
        ltol = 2e-5 if sac else TOL  # SAC's target passes through atanh(tanh(x))
        for c in range(2 if meta["twin"] else 1):
            want = out["losses"][c]
            assert abs(float(closs[c]) - want) <= ltol * max(1.0, abs(want)), (it, c)
        assert G.rel_err(t._ws["td_target"], out["target"].reshape(-1)) < ltol
        assert G.rel_err(t._ws["q1_value"], out["q1_value"]) < TOL
        if meta["twin"]:
            assert G.rel_err(t._ws["q2_value"], out["q2_value"]) < TOL
        assert G.rel_err(t._ws["td_error"], out["td_error"]) < 1e-4
    for mod, net in _oracle_modules(t, st):
        _cmp_net(mod, net, 2e-5 if (sac and mod is t.actor_network) else TOL, name)
    if sac and meta["learn_alpha"]:
        assert G.rel_err(t.log_alpha, st.log_alpha) < TOL


def _config_case(algo):
    """Config-4 (SAC) / config-5 (TD3) per-GPU shapes, B 2048, as test_actor_critic_gpu."""
    S, A, B = (256, 32, 2048) if algo == "sac" else (512, 64, 2048)
    gen = torch.Generator().manual_seed(0 if algo == "sac" else 1)
    actor = _rand_net([S, 256, 256, 2 * A if algo == "sac" else A],
                      ["relu", "relu", "linear" if algo == "sac" else "tanh"], gen)
    q1 = _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen)
    q2 = _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen)
    arrays = {}
    _net_arrays(arrays, "actor0", actor)
    _net_arrays(arrays, "q1_0", q1)
    _net_arrays(arrays, "q2_0", q2)
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             action=torch.rand(B, A, generator=gen) * 1.98 - 0.99,
             next_action=torch.zeros(B, A), reward=torch.randn(B, 1, generator=gen),
             not_terminal=(torch.rand(B, 1, generator=gen) > 0.005).float())
    meta = dict(S=S, A=A, B=B, sizes=[256, 256], acts=["relu", "relu"], twin=True, gamma=0.99,
                tau=0.005, lr=1e-3, n_updates=2)
    if algo == "sac":
        meta.update(learn_alpha=True, entropy_temperature=0.1, target_entropy=-float(A),
                    backprop=True)
        t = _build_sac(meta, arrays)
        st = O.SacState(actor, q1, q2, lr=1e-3, entropy_temperature=0.1, learn_alpha=True,
                        target_entropy=-float(A))
    else:
        meta.update(noise_variance=0.2, noise_clip=0.5, delay=2)
        t = _build_td3(meta, arrays)
        st = O.Td3State(actor, q1, q2, lr=1e-3)
    return t, st, b, meta, arrays, gen


@pytest.mark.parametrize("algo", ["sac", "td3"])
def test_weighted_update_at_config_shapes(algo):
    """Weighted updates at the config-4 / config-5 per-GPU shapes, with the bounds of
    test_sac_config4_shard_matches_oracle / test_td3_config5_shard_matches_oracle."""
    t, st, b, meta, arrays, gen = _config_case(algo)
    B, A = meta["B"], meta["A"]
    gb = _pbatch({k: v.cuda() for k, v in b.items()})
    ltol = 2e-5 if algo == "sac" else TOL
    for it in range(meta["n_updates"]):
        w = 0.05 + 0.95 * torch.rand(B, generator=gen)
        nn_, nc = torch.randn(B, A, generator=gen), torch.randn(B, A, generator=gen)
        arrays[f"noise{it}.next"], arrays[f"noise{it}.cur"] = nn_.numpy(), nc.numpy()
        _inject(t, arrays, it)
        if algo == "sac":
            out = PA.weighted_sac_update(st, b, nn_, nc, w, gamma=0.99, tau=0.005)
            crit = (t.actor_network, t.q1_network_target, t.q2_network_target, t._fill_critic)
        else:
            out = PA.weighted_td3_update(st, b, nn_, it, w, gamma=0.99, tau=0.005)
            crit = (t.actor_network_target, t.q1_network_target, t.q2_network_target, t._fill)
        if it == 0:
            t._critic_step(gb, *crit, sample_weight=w.cuda())
            # the critics the unweighted shard tests bound: q1 and q2 for SAC, q1 for TD3
            for c in ("q1", "q2") if algo == "sac" else ("q1",):
                for pi, g in enumerate(t.net_grads(getattr(t, c + "_network"))):
                    G.grad_close(g, out["grads"][c][pi], (c + " grad", pi))
            assert G.rel_err(t._ws["td_target"], out["target"].reshape(-1)) < (
                5e-5 if algo == "sac" else TOL)
        closs, aloss = t.train_batch(gb, it, importance_weights=w.cuda())
        for c in range(2):
            assert abs(float(closs[c]) - out["losses"][c]) <= ltol * max(1.0, abs(out["losses"][c]))
        if aloss is not None:
            assert abs(float(aloss[0]) - out["losses"][2]) <= ltol * max(1.0, abs(out["losses"][2]))
    for net, onet in ((t.q1_network, st.q1), (t.actor_network, st.actor)):
        for i, seq in enumerate(net.fc.dnn):
            _adam_close(seq[0].weight, onet["W"][i], meta)
    if algo == "sac":
        assert G.rel_err(t.log_alpha, st.log_alpha) < TOL
    else:
        for i, seq in enumerate(t.actor_network_target.fc.dnn):
            _adam_close(seq[0].weight, st.actor_t["W"][i], meta)


@pytest.mark.parametrize("name", SAC_CASES + TD3_CASES + ["sac_config4", "td3_config5"])
def test_td_error_and_priorities(name):
    """td_error_out is torch's max(|q1 - y|, |q2 - y|) on the kernel's own outputs, bit for bit,
    and its priorities are within 4 fp64 ulp of numpy."""
    from reagent_b200.replay_memory import PrioritizedUpdate

    if name.endswith(("config4", "config5")):
        t, _, b, meta, arrays, gen = _config_case(name[:3])
        gb = _pbatch({k: v.cuda() for k, v in b.items()})
        arrays["noise0.next"] = torch.randn(meta["B"], meta["A"], generator=gen).numpy()
        arrays["noise0.cur"] = torch.randn(meta["B"], meta["A"], generator=gen).numpy()
    else:
        t, gb, _, _, meta, arrays = _golden(name)
    _inject(t, arrays, 0)
    w = torch.rand(meta["B"], device="cuda") + 0.05
    t.train_batch(gb, 0, importance_weights=w)
    ws = t._ws
    q1, y = ws["q1_value"], ws["td_target"]
    want = (q1 - y).abs()
    if meta["twin"]:
        want = torch.maximum(want, (ws["q2_value"] - y).abs())
    assert torch.equal(ws["td_error"], want)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=1000, eps=1e-6)
    n = meta["B"]
    rng = np.random.RandomState(n)
    cap = 1 << 12
    heap, depth, _ = filled_heap(cap, rng)
    heap_d = torch.from_numpy(heap).cuda()
    idx = torch.from_numpy(rng.randint(0, cap, n).astype(np.int64)).cuda()
    p = torch.empty(n, dtype=torch.float64, device="cuda")
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    dm = torch.tensor([0.0], dtype=torch.float64, device="cuda")
    rows_update(heap_d, depth, idx, ws["td_error"], 1.0, per, p, dm, st)
    pw = PA.twin_td_priorities(q1.cpu().numpy(), ws["q2_value"].cpu().numpy() if meta["twin"]
                               else None, y.cpu().numpy(), per.alpha, per.eps)
    assert int(st[0]) == 0 and ulps(p.cpu().numpy(), pw).max() <= 4


# ---------------------------------------------------------------------------
# the online step
# ---------------------------------------------------------------------------
def _cfg(algo):
    import bench

    return dict(bench.CONFIGS[4 if algo == "sac" else 5], cap=4096, B=256)


def _bounds(cfg):
    return -np.ones(cfg["A"], np.float32), np.ones(cfg["A"], np.float32)


class _Noise:
    """Fixed device noise buffers behind the trainer's noise_hook, refilled between steps."""

    def __init__(self, t, B, A, seed):
        self.buf = {k: torch.empty(B, A, device="cuda") for k in ("next", "cur")}
        self.gen = torch.Generator().manual_seed(seed)
        t.noise_hook = lambda name, shape, device: self.buf[name]
        self.refill()

    def refill(self):
        torch.cuda.synchronize()
        for v in self.buf.values():
            v.copy_(torch.randn(v.shape, generator=self.gen))


@pytest.mark.parametrize("algo", ["sac", "td3"])
def test_online_per_loop_equals_host_replica(algo):
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedPolicyStep

    cfg = _cfg(algo)
    B = cfg["B"]
    low, high = _bounds(cfg)
    base = transition_stream(3000, 3, cfg=cfg)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=20, eps=1e-6)
    rb_d, t_d = bench_setup(cfg, base)
    rb_h, _ = bench_setup(cfg, base)

    def twin_critic_priorities(t):
        ws = t._ws
        return PA.twin_td_priorities(ws["q1_value"].cpu().numpy(), ws["q2_value"].cpu().numpy(),
                                     ws["td_target"].cpu().numpy(), per.alpha, per.eps)

    assert_matches_host_replica(
        lambda: FusedPolicyStep(t_d, rb_d, B, low, high, online=True, per=per), rb_h,
        transition_stream(40, 4, cfg=cfg), lambda rb: rb.sample_policy_network_batch(B, low, high),
        twin_critic_priorities)
    assert t_d.all_batches_processed == 31


@pytest.mark.parametrize("with_per", [False, True])
@pytest.mark.parametrize("algo", ["sac", "td3"])
def test_online_captured_equals_eager(algo, with_per):
    """The same online steps through graph replay and through eager launches of the same update
    from identical starting states, the noise from fixed buffers: losses, every network, the
    tree, the max priority and the batch counter agree bit for bit (TD3: both phases)."""
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedPolicyStep

    cfg = _cfg(algo)
    low, high = _bounds(cfg)
    base = transition_stream(3000, 7, cfg=cfg)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=10, eps=1e-6) if with_per else None

    def setup():
        rb, t = bench_setup(cfg, base)
        noise = _Noise(t, cfg["B"], cfg["A"], 11)
        random.seed(5)
        return FusedPolicyStep(t, rb, cfg["B"], low, high, online=True, per=per), noise.refill

    snap = assert_captured_equals_eager(
        setup, transition_stream(7, 8, cfg=cfg), 7,
        lambda f: [_state(f.trainer), tree(f), f.trainer.all_batches_processed],
        drop_priority=(lambda i: i % 2) if with_per else None, scalar_loss=False)
    assert snap[-1] == 8


@pytest.mark.parametrize("algo", ["sac", "td3"])
def test_online_step_equals_train_batch_on_the_drawn_indices(algo):
    """Without per: each captured step trains exactly like train_batch on
    sample_policy_network_batch(indices=...) of the indices it drew."""
    from reagent_b200.training.fused_step import FusedPolicyStep

    cfg = _cfg(algo)
    B = cfg["B"]
    low, high = _bounds(cfg)
    base = transition_stream(3000, 12, cfg=cfg)
    extra = transition_stream(3, 13, cfg=cfg)
    rb1, t1 = bench_setup(cfg, base)
    rb2, t2 = bench_setup(cfg, base)
    n1, n2 = _Noise(t1, B, cfg["A"], 21), _Noise(t2, B, cfg["A"], 21)
    random.seed(9)
    fused = FusedPolicyStep(t1, rb1, B, low, high, online=True)
    # t2 repeats the warm-up update (batch 0) on the same indices
    idx = fused._idx_buf[0].clone()
    t2.train_batch(rb2.sample_policy_network_batch(B, low, high, indices=idx), 0)
    for i in range(3):
        n1.refill()
        n2.refill()
        tr = {k: v[i] for k, v in extra.items()}
        out = fused.step(tr)
        torch.cuda.current_stream().synchronize()
        host_add(rb2, tr)
        idx = fused._idx_buf[0].clone()
        closs, _ = t2.train_batch(rb2.sample_policy_network_batch(B, low, high, indices=idx), i + 1)
        assert torch.equal(out, closs.cpu())
        assert all(torch.equal(a, b) for a, b in zip(_state(t1), _state(t2)))


@pytest.mark.parametrize("algo", ["sac", "td3"])
def test_online_per_nan_reward_raises(algo):
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedPolicyStep

    cfg = _cfg(algo)
    low, high = _bounds(cfg)
    rb, t = bench_setup(cfg, transition_stream(3000, 5, cfg=cfg))
    random.seed(1)
    fused = FusedPolicyStep(t, rb, cfg["B"], low, high, online=True, per=PrioritizedUpdate())
    assert_nan_reward_raises(fused, transition_stream(10, 6, cfg=cfg))
