"""Pins the float64 head restatements (oracle/heads_fp64.py) against oracle/td_oracle.py, which
tests/test_oracle_golden.py pins to the unmodified reference.  On every C51, QR-DQN,
ParametricDQN and CPE golden case the networks of td_oracle run in float64; the head inputs
and d loss / d head output are taken from those runs and the restatement, fed the same inputs,
must give the same loss and gradient.  CPU only."""
import pytest
import torch

from oracle import heads_fp64 as H
from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import (C51_CASES, DQN_CPE_CASES, PDQN_CASES, QRDQN_CASES, _c51_kwargs,
                                _dqn_kwargs)

TOL = 1e-5
f64 = torch.float64


@pytest.fixture(autouse=True)
def _float64_default():
    old = torch.get_default_dtype()
    torch.set_default_dtype(f64)
    yield
    torch.set_default_dtype(old)


def _to64(net):
    if net.get("kind") == "dueling":
        return {"kind": "dueling", **{k: _to64(net[k]) for k in ("shared", "adv", "val")}}
    return {"W": [w.detach().to(f64).requires_grad_(True) for w in net["W"]],
            "b": [b.detach().to(f64).requires_grad_(True) for b in net["b"]], "act": net["act"]}


def _load(name, prefixes):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    nets = {p: _to64(G.oracle_net(arrays, p, acts)) for p in prefixes}
    batch = {k: (v.to(f64) if v.is_floating_point() else v)
             for k, v in G.batch_tensors(arrays).items()}
    return meta, nets, batch


class _Taps:
    """Wraps td_oracle.mlp: records each top-level network's outputs in call order and, for
    outputs computed with autograd on, d loss / d output when the loss is differentiated."""

    def __init__(self, monkeypatch, nets):
        self.names = {id(n): k for k, n in nets.items()}
        self.out, self.grad = {}, {}
        inner = O.mlp

        def mlp(net, x):
            y = inner(net, x)
            name = self.names.get(id(net))
            if name is not None:
                outs = self.out.setdefault(name, [])
                key = (name, len(outs))
                outs.append(y.detach())
                if y.requires_grad:
                    y.register_hook(lambda g, k=key: self.grad.__setitem__(k, g.detach()))
            return y

        monkeypatch.setattr(O, "mlp", mlp)

    def last(self, name):
        """(output, d loss / d output) of the network's last evaluation: q(s) of each update."""
        i = len(self.out[name]) - 1
        return self.out[name][i], self.grad.get((name, i))

    def first(self, name):
        return self.out[name][0]


def _close(got, want, what):
    assert G.rel_err(got, want) < TOL, (what, G.rel_err(got, want))


@pytest.mark.parametrize("name", C51_CASES)
def test_c51_head_fp64_matches_oracle(name, monkeypatch):
    meta, nets, batch = _load(name, ["q0", "qt0"])
    q, qt = nets["q0"], nets["qt0"]
    kw = _c51_kwargs(meta, batch)
    taps = _Taps(monkeypatch, {"q": q, "qt": qt})
    loss = O.c51_loss(q, qt, batch, gamma=meta["gamma"], **kw)
    loss.backward()
    cur, dz = taps.last("q")  # q(s') first when double-Q selects with it, q(s) last
    N, qmin, qmax = meta["N"], meta["qmin"], meta["qmax"]
    got = H.c51_head(taps.first("q") if len(taps.out["q"]) > 1 else None, taps.first("qt"), cur,
                     batch["action"], batch["next_action"], batch["possible_next_actions_mask"],
                     batch["reward"], batch["not_terminal"], torch.linspace(qmin, qmax, N),
                     gamma=meta["gamma"], qmin=qmin, qmax=qmax,
                     scale_support=(qmax - qmin) / (N - 1.0), double_q=meta["double_q"],
                     maxq=meta["maxq"], discount_src=kw.get("discount_src"),
                     reward_boost=kw.get("reward_boost"))
    _close(got["loss"], loss.detach(), "loss")
    _close(got["loss_partials"].mean(), loss.detach(), "loss_partials")
    _close(got["dz"], dz, "dz")


@pytest.mark.parametrize("name", QRDQN_CASES)
def test_qr_head_fp64_matches_oracle(name, monkeypatch):
    meta, nets, batch = _load(name, ["q0", "qt0"])
    q, qt = nets["q0"], nets["qt0"]
    kw = dict(double_q=meta["double_q"], maxq=meta["maxq"], num_atoms=meta["N"])
    if meta["multi_steps"] is not None:
        kw["discount_src"] = batch["step"]
    taps = _Taps(monkeypatch, {"q": q, "qt": qt})
    loss, aux = O.qrdqn_loss(q, qt, batch, gamma=meta["gamma"], **kw)
    loss.backward()
    cur, dz = taps.last("q")
    N = meta["N"]
    got = H.qr_head(taps.first("q") if len(taps.out["q"]) > 1 else None, taps.first("qt"), cur,
                    batch["action"], batch["next_action"], batch["possible_next_actions_mask"],
                    batch["reward"], batch["not_terminal"], gamma=meta["gamma"], **kw,
                    row_chunk=7)  # several chunks, the last one ragged
    B = cur.shape[0]
    _close(got["loss"], loss.detach(), "loss")
    _close(got["loss_partials"].sum() / (N * B * N), loss.detach(), "loss_partials")
    _close(got["dz"], dz, "dz")
    _close(got["all_q_values"], aux["all_q"], "all_q")
    if meta["maxq"]:
        assert torch.equal(got["next_action_idx"], aux["next_action"].reshape(-1))


@pytest.mark.parametrize("name", PDQN_CASES)
def test_pdqn_head_fp64_matches_oracle(name, monkeypatch):
    meta, nets, batch = _load(name, ["q0", "qt0"])
    q, qt = nets["q0"], nets["qt0"]
    taps = _Taps(monkeypatch, {"q": q, "qt": qt})
    discount_src = batch["step"] if meta["multi_steps"] is not None else None
    td, _, _ = O.pdqn_update(q, qt, O.AdamState(O.net_params(q)), batch, gamma=meta["gamma"],
                             tau=meta["tau"], double_q=meta["double_q"], maxq=meta["maxq"],
                             loss=meta["loss"], discount_src=discount_src)
    cur, dz = taps.last("q")  # q on the tiled next actions first (maxq), q(s, a) last
    B = cur.shape[0]
    M = batch["possible_next_actions"].shape[0] // B if meta["maxq"] else 0
    got = H.pdqn_head(taps.first("q") if M else None, taps.first("qt"),
                      batch["possible_next_actions_mask"] if M else None, batch["reward"],
                      batch["not_terminal"], cur, max_num_action=M, gamma=meta["gamma"],
                      double_q=meta["double_q"], loss=meta["loss"], discount_src=discount_src)
    _close(got["loss"], td, "loss")
    _close(got["dz"], dz.reshape(-1), "dz")


@pytest.mark.parametrize("name", DQN_CPE_CASES)
def test_cpe_heads_fp64_matches_oracle(name, monkeypatch):
    meta, nets, batch = _load(name, ["q0", "r0", "c0", "ct0"])
    taps = _Taps(monkeypatch, {"q": nets["q0"], "r": nets["r0"], "c": nets["c0"], "ct": nets["ct0"]})
    kw = _dqn_kwargs(meta, batch)
    rl, cl, prop = O.dqn_cpe_losses(nets["q0"], nets["r0"], nets["c0"], nets["ct0"], batch,
                                    gamma=meta["gamma"], temperature=meta["temperature"],
                                    num_actions=meta["A"], maxq=meta["maxq"], loss=meta["loss"],
                                    discount_src=kw.get("discount_src"))
    (rl + cl).backward()
    mrc = batch["reward"]
    if batch["metrics"].shape[1] > 0:
        mrc = torch.cat((batch["reward"], batch["metrics"]), dim=1)
    mask = batch["possible_next_actions_mask"] if meta["maxq"] else batch["next_action"]
    (r_est, dz_r), (qc, dz_c) = taps.last("r"), taps.last("c")
    got = H.cpe_heads(taps.first("q"), mask, batch["action"], mrc, batch["not_terminal"], r_est, qc,
                      taps.first("ct"), temperature=meta["temperature"], gamma=meta["gamma"],
                      loss=meta["loss"], discount_src=kw.get("discount_src"))
    _close(got["loss"], torch.stack([rl.detach(), cl.detach()]), "losses")
    _close(got["propensities_next"], prop, "propensities")
    _close(got["dz_reward"], dz_r, "dz_reward")
    _close(got["dz_qcpe"], dz_c, "dz_qcpe")


def test_dueling_fold_fp64_matches_oracle_forward():
    """The folded Linear on [h_adv | h_val] reproduces td_oracle's dueling forward (with atoms)
    on the qrdqn_dueling golden, and the unfold is the vector-Jacobian product of that forward."""
    meta, nets, batch = _load("qrdqn_dueling", ["q0"])
    q = nets["q0"]
    A, N = meta["A"], meta["N"]
    shared = O.mlp(q["shared"], batch["state"])
    h_adv = O.mlp({**q["adv"], "W": q["adv"]["W"][:-1], "b": q["adv"]["b"][:-1]}, shared)
    h_val = O.mlp({**q["val"], "W": q["val"]["W"][:-1], "b": q["val"]["b"][:-1]}, shared)
    p = [q["adv"]["W"][-1], q["adv"]["b"][-1], q["val"]["W"][-1], q["val"]["b"][-1]]
    W_q, b_q = H.dueling_fold(*[t.detach() for t in p], A, N)
    want = O.mlp(q, batch["state"])
    _close(torch.cat([h_adv, h_val], 1).detach() @ W_q.t() + b_q, want.detach(), "fold")
    # unfold: d(sum q * R) / d true params, R random, against autograd of td_oracle's forward
    gen = torch.Generator().manual_seed(0)
    Rw = torch.randn(want.shape, generator=gen, dtype=f64)
    gw = torch.autograd.grad((want * Rw).sum(), p)
    h = torch.cat([h_adv, h_val], 1).detach()
    got = H.dueling_unfold(*p, Rw.t() @ h, Rw.sum(0), A, N)
    for g, w, what in zip(got, gw, ("dW_adv", "db_adv", "dW_val", "db_val")):
        _close(g, w, what)
