"""Pins the CPU restatement (oracle/td_oracle.py) against golden vectors produced by the
UNMODIFIED reference (oracle/make_golden.py).  CPU only."""
import pytest
import torch

from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import (C51_CASES, DQN_CASES, DQN_CPE_CASES, PDQN_CASES, QRDQN_CASES,
                                SAC_CASES, TD3_CASES, _c51_kwargs, _dqn_kwargs)
from tests.golden_util import _cmp_losses, _cmp_net


@pytest.mark.parametrize("name", DQN_CASES)
def test_dqn_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = _dqn_kwargs(meta, batch)
    for it in range(meta["n_updates"]):
        loss, grads, aux = O.dqn_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6
            assert G.rel_err(aux["all_q"], arrays["all_q0"]) < 1e-6
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6
            assert G.rel_err(ps[2 * i + 1], b) < 1e-6


# ---------------------------------------------------------------------------
# replay sampler restatement vs the reference buffers
# ---------------------------------------------------------------------------
REPLAY_CASES = ["replay_uniform_h1", "replay_uniform_h3_wrap", "replay_uniform_h5_cont",
                "replay_per_h1", "replay_per_h3_wrap_zero", "replay_per_big"]


@pytest.mark.parametrize("name", REPLAY_CASES)
def test_replay_oracle_matches_reference(name):
    import random

    import numpy as np

    from oracle.replay_oracle import ReplayOracle

    arrays, meta = G.load(name)
    rb = ReplayOracle(meta["cap"], meta["horizon"], meta["gamma"], meta["prioritized"])
    keys = meta["keys"]
    for t in range(meta["n_add"]):
        rb.add(**{k: arrays[f"stream.{k}"][t] for k in keys})
    assert np.array_equal(rb.valid, arrays["valid"])
    random.seed(meta["seed"] + 100)
    torch.manual_seed(meta["seed"] + 100)
    for s_i in range(meta["n_samples"]):
        out = rb.sample_transition_batch(meta["B"])
        for f, v in out.items():
            key = f"sample{s_i}.{f}"
            if key not in arrays:
                continue
            want = arrays[key]
            got = np.asarray(v).reshape(want.shape)
            if f.startswith("next_"):
                # "When the transition is terminal next_state_batch has undefined contents"
                # (circular_replay_buffer.py:621): the reference may read np.empty() memory.
                keep = ~arrays[f"sample{s_i}.terminal"].reshape(-1)
                got, want = got[keep], want[keep]
            assert np.array_equal(got, want), key


# ---------------------------------------------------------------------------
# SAC / TD3 restatements vs the reference trainers
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("name", SAC_CASES)
def test_sac_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    actor = G.oracle_net(arrays, "actor0", acts)
    q1 = G.oracle_net(arrays, "q1_0", acts)
    q2 = G.oracle_net(arrays, "q2_0", acts) if meta["twin"] else None
    st = O.SacState(actor, q1, q2, lr=meta["lr"], entropy_temperature=meta["entropy_temperature"],
                    learn_alpha=meta["learn_alpha"], target_entropy=meta["target_entropy"])
    batch = G.batch_tensors(arrays)
    for it in range(meta["n_updates"]):
        out = O.sac_update(st, batch, torch.from_numpy(arrays[f"noise{it}.next"]),
                           torch.from_numpy(arrays[f"noise{it}.cur"]), gamma=meta["gamma"],
                           tau=meta["tau"], backprop_through_log_prob=meta["backprop"])
        _cmp_losses(out["losses"], arrays["losses"][it], 2e-6)
        if it == 0:
            names = ["q1"] + (["q2"] if meta["twin"] else []) + ["actor"] + (
                ["alpha"] if meta["learn_alpha"] else [])
            for oi, nm in enumerate(names):
                for pi, g in enumerate(out["grads"][nm]):
                    assert G.rel_err(g, arrays[f"grad0.opt{oi}.{pi}"]) < 2e-5, (nm, pi)
    _cmp_net(st.actor, arrays, "actorN", 1e-5)
    _cmp_net(st.q1, arrays, "q1_N", 1e-5)
    _cmp_net(st.q1t, arrays, "q1t_N", 1e-5)
    if meta["twin"]:
        _cmp_net(st.q2, arrays, "q2_N", 1e-5)
        _cmp_net(st.q2t, arrays, "q2t_N", 1e-5)
    if meta["learn_alpha"]:
        assert G.rel_err(st.log_alpha, arrays["log_alpha_N"]) < 1e-6


@pytest.mark.parametrize("name", TD3_CASES)
def test_td3_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    actor = G.oracle_net(arrays, "actor0", meta["acts"] + ["tanh"])
    cacts = meta["acts"] + ["linear"]
    q1 = G.oracle_net(arrays, "q1_0", cacts)
    q2 = G.oracle_net(arrays, "q2_0", cacts) if meta["twin"] else None
    st = O.Td3State(actor, q1, q2, lr=meta["lr"])
    batch = G.batch_tensors(arrays)
    for it in range(meta["n_updates"]):
        out = O.td3_update(st, batch, torch.from_numpy(arrays[f"noise{it}.next"]), it,
                           gamma=meta["gamma"], tau=meta["tau"],
                           noise_variance=meta["noise_variance"], noise_clip=meta["noise_clip"],
                           delayed_policy_update=meta["delay"])
        _cmp_losses(out["losses"], arrays["losses"][it], 2e-6)
    _cmp_net(st.actor, arrays, "actorN", 1e-5)
    _cmp_net(st.actor_t, arrays, "actort_N", 1e-5)
    _cmp_net(st.q1, arrays, "q1_N", 1e-5)
    _cmp_net(st.q1t, arrays, "q1t_N", 1e-5)
    if meta["twin"]:
        _cmp_net(st.q2, arrays, "q2_N", 1e-5)
        _cmp_net(st.q2t, arrays, "q2t_N", 1e-5)


# oracle-only for now: the dueling quantile head has no CUDA path yet (SURVEY M6 / config 3 note)
QRDQN_ORACLE_ONLY = []


@pytest.mark.parametrize("name", QRDQN_CASES + QRDQN_ORACLE_ONLY)
def test_qrdqn_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = dict(double_q=meta["double_q"], maxq=meta["maxq"], num_atoms=meta["N"])
    if meta["multi_steps"] is not None:
        kw["discount_src"] = batch["step"]
    for it in range(meta["n_updates"]):
        loss, grads, aux = O.qrdqn_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6
            assert G.rel_err(ps[2 * i + 1], b) < 1e-6

@pytest.mark.parametrize("horizon,n", [(1, 512), (3, 512), (2, 300)])
def test_replay_oracle_bulk_fill_equals_sequential_adds(horizon, n):
    """ReplayOracle.bulk_fill (used by the config-2-size GPU test and the CPU baseline of
    bench.py) leaves exactly the state of n sequential add() calls: validity, storage and the
    fp64 sum tree bit for bit (sequential delta propagation, sum_tree.py:164-189)."""
    import numpy as np

    from oracle.replay_oracle import ReplayOracle

    rng = np.random.RandomState(horizon * 100 + n)
    cap = 512
    st = dict(observation=rng.randn(n, 4).astype(np.float32),
              action=rng.randint(0, 3, n).astype(np.int64),
              reward=rng.randn(n).astype(np.float32), terminal=rng.rand(n) < 0.05,
              priority=rng.uniform(0.1, 10, n))
    a = ReplayOracle(cap, update_horizon=horizon, prioritized=True)
    b = ReplayOracle(cap, update_horizon=horizon, prioritized=True)
    for t in range(n):
        a.add(**{k: v[t] for k, v in st.items()})
    b.bulk_fill(st)
    assert np.array_equal(a.valid, b.valid)
    for x, y in zip(a.tree.nodes, b.tree.nodes):
        assert np.array_equal(x, y)
    assert (a.ep, a.add_count) == (b.ep, b.add_count)
    assert a.tree.max_recorded_priority == b.tree.max_recorded_priority
    for k in a.store:
        assert np.array_equal(a.store[k], b.store[k])


@pytest.mark.parametrize("name", ["inputmaker_dqn_uniform", "inputmaker_dqn_per_masks",
                                  "inputmaker_policy_uniform", "inputmaker_policy_per_h3"])
def test_replay_oracle_plus_inputmaker_formulas_match_reference(name):
    """The oracle sampler followed by the InputMaker arithmetic (one-hot, zeroed terminal
    next-actions, 1 - terminal, affine action rescale: trainer_preprocessor.py:72-227,
    training/utils.py:13-29) reproduces the reference InputMakers' outputs on the same seeds --
    this is what the config-2-size GPU test compares the fused kernel with."""
    import random

    import numpy as np

    from oracle.replay_oracle import ReplayOracle

    arrays, meta = G.load(name)
    ro = ReplayOracle(meta["cap"], update_horizon=meta["horizon"], gamma=meta["gamma"],
                      prioritized=meta["prioritized"])
    st = {k: arrays[f"stream.{k}"] for k in meta["keys"]}
    for t in range(meta["n_add"]):
        ro.add(**{k: v[t] for k, v in st.items()})
    random.seed(meta["seed"] + 200)
    torch.manual_seed(meta["seed"] + 200)
    A = meta["A"]
    for s_i in range(meta["n_samples"]):
        ob = ro.sample_transition_batch(meta["B"])
        pre = f"sample{s_i}."
        assert np.array_equal(ob["indices"], arrays[pre + "indices"].reshape(-1))
        term = ob["terminal"].astype(bool)
        assert np.array_equal(term, arrays[pre + "terminal"].reshape(-1))
        assert np.array_equal(ob["state"], arrays[pre + "state"])
        assert np.array_equal(ob["next_state"][~term], arrays[pre + "next_state"][~term])
        np.testing.assert_allclose(ob["reward"], arrays[pre + "reward"].reshape(-1), rtol=2e-6, atol=1e-6)
        assert np.array_equal(1.0 - term.astype(np.float32), arrays[pre + "not_terminal"].reshape(-1))
        if meta["continuous"]:
            lo, hi = arrays["action_low"], arrays["action_high"]
            resc = lambda a: ((a - lo) / (hi - lo)) * np.float32(2.0) + np.float32(-1.0)
            assert np.array_equal(resc(ob["action"]).astype(np.float32), arrays[pre + "action"])
            na = resc(ob["next_action"]).astype(np.float32) * (~term)[:, None]
            assert np.array_equal(na, arrays[pre + "next_action"])
        else:
            eye = np.eye(A, dtype=np.float32)
            assert np.array_equal(eye[ob["action"]], arrays[pre + "action"])
            assert np.array_equal(eye[ob["next_action"]] * (~term)[:, None], arrays[pre + "next_action"])


@pytest.mark.parametrize("name", DQN_CPE_CASES)
def test_dqn_cpe_oracle_matches_reference(name):
    """CPE heads (dqn_trainer_base.py:332-452): the oracle's reward / CPE q-value losses,
    gradients and post-update networks against the unmodified reference DQNTrainer with
    calc_cpe_in_training=True."""
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    rn = G.oracle_net(arrays, "r0", acts, requires_grad=True)
    qc = G.oracle_net(arrays, "c0", acts, requires_grad=True)
    qct = G.oracle_net(arrays, "ct0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    adam_r = O.AdamState(O.net_params(rn), lr=meta["lr"])
    adam_c = O.AdamState(O.net_params(qc), lr=meta["lr"])
    kw = _dqn_kwargs(meta, batch)
    ckw = dict(gamma=meta["gamma"], temperature=meta["temperature"], num_actions=meta["A"],
               maxq=meta["maxq"], loss=meta["loss"], discount_src=kw.get("discount_src"))
    for it in range(meta["n_updates"]):
        loss, grads, aux = O.dqn_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"], **kw)
        rl, cl, gr, gc = O.dqn_cpe_update(q, rn, adam_r, qc, qct, adam_c, batch, tau=meta["tau"], **ckw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        for got, want in ((rl, arrays["cpe_losses"][it][0]), (cl, arrays["cpe_losses"][it][1])):
            assert abs(got - want) <= 1e-6 * max(1.0, abs(want)), (it, got, want)
        if it == 0:
            for i, g in enumerate(gr):
                assert G.rel_err(g, arrays[f"grad0r.{i}"]) < 1e-6
            for i, g in enumerate(gc):
                assert G.rel_err(g, arrays[f"grad0c.{i}"]) < 1e-6
    for net, prefix in ((q, "qN"), (qt, "qtN"), (rn, "rN"), (qc, "cN"), (qct, "ctN")):
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], b) < 1e-6, (prefix, i)


@pytest.mark.parametrize("name", PDQN_CASES)
def test_pdqn_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    rn = G.oracle_net(arrays, "r0", acts, requires_grad=True) if meta["with_reward_net"] else None
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    adam_r = O.AdamState(O.net_params(rn), lr=meta["lr"]) if rn is not None else None
    kw = dict(double_q=meta["double_q"], maxq=meta["maxq"], loss=meta["loss"], reward_net=rn, adam_r=adam_r,
              discount_src=batch["step"] if meta["multi_steps"] is not None else None)
    for it in range(meta["n_updates"]):
        td, rl, grads = O.pdqn_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(td - arrays["losses"][it][0]) <= 1e-6 * max(1.0, abs(arrays["losses"][it][0]))
        if rn is not None:
            assert abs(rl - arrays["losses"][it][1]) <= 1e-6 * max(1.0, abs(arrays["losses"][it][1]))
        if it == 0:
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6
    nets = [(q, "qN"), (qt, "qtN")] + ([(rn, "rN")] if rn is not None else [])
    for net, prefix in nets:
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6 and G.rel_err(ps[2 * i + 1], b) < 1e-6, (prefix, i)


@pytest.mark.parametrize("name", C51_CASES)
def test_c51_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = _c51_kwargs(meta, batch)
    for it in range(meta["n_updates"]):
        loss, grads = O.c51_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6 and G.rel_err(ps[2 * i + 1], b) < 1e-6, (prefix, i)
