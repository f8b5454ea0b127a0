"""GPU parity of the QR-DQN update (fused trunk + 2-D tiled head + distributional head kernel)
vs golden vectors from the unmodified reference QRDQNTrainer and vs the CPU oracle at a
config-3-shaped size (A=32, N=200 atoms)."""
import pytest
import torch

from oracle import td_oracle as O
from tests import golden_util as G
from tests.builders import _batch, _build_qr
from tests.golden_cases import QRDQN_CASES

pytestmark = pytest.mark.gpu
TOL = 1e-5


@pytest.mark.parametrize("name", QRDQN_CASES)
@pytest.mark.parametrize("fast", [False, True])
def test_qrdqn_matches_reference(name, fast):
    from reagent_b200.training import run_update

    arrays, meta = G.load(name)
    t = _build_qr(meta, arrays)
    batch = _batch(G.batch_tensors(arrays, "cuda"), meta)
    for it in range(meta["n_updates"]):
        ref = arrays["losses"][it]
        if fast:
            loss = float(t.train_batch(batch, it))
        elif it == 0:
            opts = t.optimizers()
            l0 = t.training_step(batch, it, 0)
            for i, g in enumerate(t.q_network_grads()):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < TOL, f"grad {i}"
            opts[0].zero_grad(); l0.backward(); opts[0].step()
            l1 = t.training_step(batch, it, 1)
            opts[1].zero_grad(); l1.backward(); opts[1].step()
            loss = float(l0.detach())
        else:
            loss = float(run_update(t, batch, it)[0].detach())
        assert abs(loss - ref) <= TOL * max(1.0, abs(ref)), (it, loss, ref)
    for net, prefix in ((t.q_network, "qN"), (t.q_network_target, "qtN")):
        ps = list(net.parameters())  # dueling: shared, advantage, value (reference order)
        pairs = G.net_pairs(arrays, prefix)
        assert len(ps) == 2 * len(pairs)
        for i, (w, b) in enumerate(pairs):
            assert G.rel_err(ps[2 * i], w) < TOL, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], b) < TOL, (prefix, i)


def test_dueling_quantile_forward_matches_reference():
    """DuelingQNetwork with atoms: (B, A, N) output, mean over actions AND atoms
    (dueling_q_network.py:92-103); the manager default is DuelingQuantile as in the reference."""
    from reagent_b200.core import types as rlt
    from reagent_b200.model_managers import DiscreteQRDQN
    from reagent_b200.net_builder import DuelingQuantile

    arrays, meta = G.load("qrdqn_dueling")
    t = _build_qr(meta, arrays)
    x = rlt.FeatureData(torch.from_numpy(arrays["batch.state"]).cuda())
    out = t.q_network(x)
    B, A, N = meta["B"], meta["A"], meta["N"]
    assert out.shape == (B, A, N)
    value, raw_adv, adv, qv = t.q_network._get_values(x)
    assert value.shape == (B, 1, N) and raw_adv.shape == (B, A, N)
    assert G.rel_err(qv, out) < TOL
    assert float(adv.mean(dim=(1, 2)).abs().max()) < 1e-6
    # against the oracle's dueling forward (pinned to the reference by tests/test_oracle_golden.py)
    qo = G.oracle_net(arrays, "q0", meta["acts"] + ["linear"])
    want = O.mlp(qo, torch.from_numpy(arrays["batch.state"]))
    assert G.rel_err(out.reshape(B, -1), want) < TOL
    assert isinstance(DiscreteQRDQN(actions=["0", "1"]).net_builder, DuelingQuantile)


def _qrdqn_oracle_chunked(qo, qt, b, *, gamma, num_atoms, chunk=256):
    """qrdqn_loss over row chunks: the loss is a mean over (N, B, N), i.e. a mean over rows of
    row-local terms, so loss = sum_c (B_c / B) * loss_c and likewise for the gradients.  Keeps
    the oracle's (N, B_c, N) tensor at 41 MB instead of 655 MB."""
    params = O.net_params(qo)
    B = b["reward"].shape[0]
    total, grads = 0.0, [torch.zeros_like(p) for p in params]
    next_action, all_q = [], []
    for r0 in range(0, B, chunk):
        sub = {k: (v[r0:r0 + chunk] if v is not None else None) for k, v in b.items()}
        lc, aux = O.qrdqn_loss(qo, qt, sub, gamma=gamma, num_atoms=num_atoms)
        w = sub["reward"].shape[0] / B
        for g, gc in zip(grads, torch.autograd.grad(lc, params)):
            g.add_(gc, alpha=w)
        total += float(lc.detach()) * w
        next_action.append(aux["next_action"])
        all_q.append(aux["all_q"])
    return total, grads, torch.cat(next_action), torch.cat(all_q)


def test_qrdqn_config3_full_batch_matches_chunked_oracle():
    """BASELINE config 3 at its real batch size: S=128, A=32, N=200, B=4096."""
    S, A, N, B = 128, 32, 200, 4096
    meta = dict(S=S, A=A, N=N, B=B, sizes=[256, 128], acts=["relu", "relu"], gamma=0.99,
                tau=0.005, maxq=True, multi_steps=None, double_q=True, lr=1e-3, n_updates=1)
    gen = torch.Generator().manual_seed(1)
    q = O.make_net([S, 256, 128, A * N], ["relu", "relu", "linear"], gen)
    qt = O.clone_net(q)
    for w in qt["W"]:
        w.add_(torch.randn(w.shape, generator=gen) * 0.02)
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = q["W"][i].numpy().copy(), q["b"][i].numpy().copy()
        arrays[f"qt0.W{i}"], arrays[f"qt0.b{i}"] = qt["W"][i].numpy().copy(), qt["b"][i].numpy().copy()
    act = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.05).float()
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen), time_diff=torch.ones(B, 1), step=None,
             not_terminal=nt, action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    t = _build_qr(meta, arrays)
    qo = O.clone_net(q, requires_grad=True)
    lo, grads, next_action, all_q = _qrdqn_oracle_chunked(qo, qt, b, gamma=0.99, num_atoms=N)
    gb = _batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    loss = float(t._qr_step(gb))
    assert abs(loss - lo) <= TOL * max(1.0, abs(lo)), (loss, lo)
    # arg max over the mean of 200 atoms: rows whose two best actions are within fp32 noise
    # may legitimately differ; they are counted, not ignored
    diff = int((t._ws["next_idx"].cpu().long() != next_action).sum())
    assert diff <= 2, diff
    assert G.rel_err(t._ws["all_q"], all_q) < TOL
    for i, g in enumerate(t.q_network_grads()):
        G.grad_close(g, grads[i], f"grad {i}")


def test_qrdqn_config3_shape_matches_oracle():
    """BASELINE config 3 network (128 -> 256 -> 128 -> 32*200) at B=256 (the oracle's (N,B,N)
    tensor at B=4096 is 655 MB; the row-local kernels do not depend on B)."""
    S, A, N, B = 128, 32, 200, 256
    meta = dict(S=S, A=A, N=N, B=B, sizes=[256, 128], acts=["relu", "relu"], gamma=0.99,
                tau=0.005, maxq=True, multi_steps=None, double_q=True, lr=1e-3, n_updates=1)
    gen = torch.Generator().manual_seed(0)
    q = O.make_net([S, 256, 128, A * N], ["relu", "relu", "linear"], gen)
    qt = O.clone_net(q)
    for w in qt["W"]:
        w.add_(torch.randn(w.shape, generator=gen) * 0.02)
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = q["W"][i].numpy().copy(), q["b"][i].numpy().copy()
        arrays[f"qt0.W{i}"], arrays[f"qt0.b{i}"] = qt["W"][i].numpy().copy(), qt["b"][i].numpy().copy()
    act = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.05).float()
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen), time_diff=torch.ones(B, 1), step=None,
             not_terminal=nt, action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    t = _build_qr(meta, arrays)
    qo = O.clone_net(q, requires_grad=True)
    qt_before = O.clone_net(qt)
    adam = O.AdamState(O.net_params(qo), lr=1e-3)
    lo, grads, aux = O.qrdqn_update(qo, qt, adam, b, gamma=0.99, tau=0.005, num_atoms=N)
    gb = _batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    loss = float(t._qr_step(gb))
    assert abs(loss - lo) <= TOL * max(1.0, abs(lo)), (loss, lo)
    assert torch.equal(t._ws["next_idx"].cpu().long(), aux["next_action"])
    assert G.rel_err(t._ws["all_q"], aux["all_q"]) < TOL
    for i, g in enumerate(t.q_network_grads()):
        G.grad_close(g, grads[i], f"grad {i}")
    # the model's own forward (act-time path, wide head) agrees with torch
    from reagent_b200.core import types as rlt
    out = t.q_network_target(rlt.FeatureData(gb.state.float_features))
    assert out.shape == (B, A, N)
    assert G.rel_err(out.reshape(B, -1), O.mlp(qt_before, b["state"])) < TOL
