"""The gate-level LSTM oracle (oracle/lstm_fp64.py) in fp64, without a GPU: its outputs are
mdnrnn_oracle.forward's and seq2reward_oracle.hidden_states' bit for bit, agree with
torch.nn.LSTM, and the weight gradients rebuilt from its dGates are autograd's."""
import pytest
import torch
import torch.nn.functional as F

from oracle import lstm_fp64 as LO
from oracle import mdnrnn_oracle as mo
from oracle import seq2reward_oracle as so

SHAPES = [(1, 1), (1, 4), (33, 1), (33, 4)]  # (H, L)


def _mdn_case(H, L, T=5, B=3, S=4, A=2, G=3, seed=0):
    params = [p.double().requires_grad_(True) for p in mo.initial_params(seed, S, A, H, L, G)]
    g = torch.Generator().manual_seed(seed + 1)
    b = dict(state=torch.randn(T, B, S, generator=g, dtype=torch.float64),
             action=F.one_hot(torch.randint(A, (T, B), generator=g), A).double(),
             next_state=torch.randn(T, B, S, generator=g, dtype=torch.float64),
             reward=torch.randn(T, B, generator=g, dtype=torch.float64),
             not_terminal=(torch.rand(T, B, generator=g) > 0.3).double())
    return params, b


def _s2r_case(H, L, T=5, B=3, S=4, A=3, seed=0):
    params = [p.double().requires_grad_(True) for p in so.initial_params(seed, S, A, H, L)]
    g = torch.Generator().manual_seed(seed + 1)
    state0 = torch.randn(B, S, generator=g, dtype=torch.float64)
    action = F.one_hot(torch.randint(A, (T, B), generator=g), A).double()
    reward = torch.randn(T, B, generator=g, dtype=torch.float64)
    valid = torch.randint(1, T + 1, (B,), generator=g)
    return params, state0, action, reward, valid


def _torch_lstm(params, x, L, h0=None):
    H = params[1].shape[1]
    rnn = torch.nn.LSTM(x.shape[2], H, L).double()
    with torch.no_grad():
        for p, q in zip(rnn.parameters(), params[:4 * L]):
            p.copy_(q)
    B = x.shape[1]
    h = torch.zeros(L, B, H, dtype=torch.float64) if h0 is None else h0.expand(L, B, H)
    y, (hn, cn) = rnn(x, (h, torch.zeros(L, B, H, dtype=torch.float64)))
    return y, hn, cn


@pytest.mark.parametrize("H,L", SHAPES)
def test_mdnrnn_wrapper_is_mdnrnn_oracle_bit_for_bit(H, L):
    params, b = _mdn_case(H, L)
    out = LO.mdnrnn(params, b["state"], b["action"], L, 3)
    ref = mo.forward(params, b["state"], b["action"], L, 3)
    for k, v in ref.items():
        assert torch.equal(out[k], v), k
    assert torch.equal(out["x"], torch.cat([b["action"], b["state"]], -1))
    assert torch.equal(out["hs"][:, 0], torch.zeros_like(out["hs"][:, 0]))
    assert torch.equal(out["cs"][:, 0], torch.zeros_like(out["cs"][:, 0]))
    assert out["hs"].shape == (L, 6, 3, H) and out["acts"].shape == (L, 5, 3, 4 * H)


@pytest.mark.parametrize("H,L", SHAPES)
def test_seq2reward_wrapper_is_seq2reward_oracle_bit_for_bit(H, L):
    params, s0, act, reward, valid = _s2r_case(H, L)
    out = LO.seq2reward(params, s0, act, L, valid)
    assert torch.equal(out["top"], so.hidden_states(params, s0, act, L))
    assert torch.equal(out["acc_reward"], so.forward(params, s0, act, L, valid))
    for l in range(L):
        assert torch.equal(out["hs"][l, 0], out["h0"])
    assert torch.equal(out["cs"][:, 0], torch.zeros_like(out["cs"][:, 0]))


@pytest.mark.parametrize("H,L", SHAPES)
@torch.no_grad()
def test_agrees_with_torch_lstm(H, L):
    params, b = _mdn_case(H, L)
    out = LO.mdnrnn(params, b["state"], b["action"], L, 3)
    y, hn, cn = _torch_lstm(params, out["x"].detach(), L)
    assert float((out["top"] - y).abs().max()) < 1e-12
    assert float((out["hs"][:, -1] - hn).abs().max()) < 1e-12
    assert float((out["cs"][:, -1] - cn).abs().max()) < 1e-12
    params, s0, act, _, _ = _s2r_case(H, L)
    out = LO.seq2reward(params, s0, act, L)
    y, hn, cn = _torch_lstm(params, act, L, out["h0"].detach())
    assert float((out["top"] - y).abs().max()) < 1e-12
    assert float((out["cs"][:, -1] - cn).abs().max()) < 1e-12
    # the gate activations are the cell's: c_t = f c_{t-1} + i g and h_t = o tanh(c_t)
    a = out["acts"]
    i, f, g, o = a.chunk(4, dim=-1)
    assert torch.allclose(out["cs"][:, 1:], f * out["cs"][:, :-1] + i * g, rtol=0, atol=1e-15)
    assert torch.allclose(out["hs"][:, 1:], o * torch.tanh(out["cs"][:, 1:]), rtol=0, atol=1e-15)


def _close(got, want, what):
    got, want = got.detach(), want.detach()
    err = float((got - want).abs().max()) / (float(want.abs().max()) + 1e-300)
    assert err < 1e-12, (what, err)


@pytest.mark.parametrize("fit_last", [False, True])
@pytest.mark.parametrize("H,L", SHAPES)
def test_mdnrnn_dgates_rebuild_the_weight_gradients(H, L, fit_last):
    params, b = _mdn_case(H, L)
    out = LO.mdnrnn(params, b["state"], b["action"], L, 3)
    ls = mo.losses(out, b["next_state"], b["reward"], b["not_terminal"], reward_weight=0.5,
                   not_terminal_weight=2.0, fit_only_one_next_step=fit_last, state_dim=4)
    ls["loss"].backward()
    dg = LO.dgates(out)
    assert dg.shape == out["acts"].shape
    assert float(dg[:, -1].abs().max()) > 0
    for i, (g, p) in enumerate(zip(LO.input_weight_grads(out, out["x"].detach(), L), params)):
        _close(g, p.grad, f"grad.{i}")


@pytest.mark.parametrize("H,L", SHAPES)
def test_seq2reward_dgates_and_dh0_rebuild_the_gradients(H, L):
    params, s0, act, reward, valid = _s2r_case(H, L)
    out = LO.seq2reward(params, s0, act, L, valid)
    loss = F.mse_loss(out["acc_reward"], so.target(reward, valid, 1.0).double())
    loss.backward()
    dg = LO.dgates(out)
    # nothing at or after a row's valid step reaches the loss
    for b_, v in enumerate(valid.tolist()):
        assert torch.equal(dg[:, v:, b_], torch.zeros_like(dg[:, v:, b_]))
    for i, (g, p) in enumerate(zip(LO.input_weight_grads(out, act, L), params)):
        _close(g, p.grad, f"grad.{i}")
    # map_linear through h0: dW_map = dh0^T state0, db_map = sum dh0
    dh0 = out["h0"].grad
    _close(dh0.T @ s0, params[4 * L + 2].grad, "map_linear.weight")
    _close(dh0.sum(0), params[4 * L + 3].grad, "map_linear.bias")
    # dh0 is the sum over layers of dL/dh_{-1}: the recurrent products of step 0
    per_layer = sum(dg[l, 0] @ params[4 * l + 1] for l in range(L))
    _close(dh0, per_layer, "dh0")
