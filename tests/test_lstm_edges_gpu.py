"""The row-tile LSTM (csrc/rb200_lstm.cuh) through its two training users, the MDN-RNN
(csrc/rb200_mdnrnn.cu) and Seq2Reward (csrc/rb200_seq2reward.cu), against the gate-level fp64
oracle (oracle/lstm_fp64.py) at the edges of the shapes they accept.

* Every launch writes into buffers filled with NaN after the workspace was allocated (the
  training workspace and the gradient partials), so a row, step or gate a kernel never writes
  cannot pass: everything the kernels promise to write must come back finite.
* Every intermediate the kernels keep is compared, not only the outputs: h and c of every
  layer and slot, the gate activations, dL/dy, dGates of every layer and step, dh0 and every
  parameter gradient.
* Each row is compared on the scale of the terms behind it.  A forward value carries the
  rounding of every product that fed it: `_fwd_env` is, per step and row, the largest sum of
  magnitudes |W||h| + |b| behind any gate pre-activation at that step or before, in any layer.
  The head adds |W_gmm||h| and the error of h carried through |W_gmm|.  A backward value is
  compared with the largest gradient at its step or any later one of its row (the recurrence
  carries the later steps' errors back), `_bwd_env`.
* The case ids name the edge each case hits: H 1 and 3 inside one MMA column tile, H 33 over
  two 32-wide k chunks (the forward's k rotation differs between CTAs), 4H = 256 and 260, the
  NG chunk edges 256 / 257 and the limit 1024, G 32 with every lane of the mixture warp live,
  the two worst shared-memory shapes, B around the 16-row tile and over two waves of one CTA
  per SM, and T = 64 for backpropagation through time.
Measured errors are appended to $RB200_TEST_RECORD_DIR/test_measurements.jsonl when that
directory exists."""
import pytest
import torch
import torch.nn.functional as F

from oracle import lstm_fp64 as LO
from oracle import mdnrnn_oracle as mo
from oracle import seq2reward_oracle as so
from reagent_b200 import _lib
from reagent_b200.core import types as rlt
from reagent_b200.core.parameters import MDNRNNTrainerParameters
from reagent_b200.evaluation import FeatureImportanceEvaluator, FeatureSensitivityEvaluator
from reagent_b200.models import MemoryNetwork, Seq2RewardNetwork
from reagent_b200.models.seq2reward_model import backward_wgrad
from reagent_b200.models.seq2reward_model import run_forward as s2r_forward
from reagent_b200.training import MDNRNNTrainer
from reagent_b200.training.workspace import ensure_gpart, param_grads
from tests.builders import _record
from tests.kernel_util import NAN, NUM_SMS

pytestmark = pytest.mark.gpu

ROWS = _lib.MDNRNN_ROWS_PER_BLOCK          # rows of one CTA
B_WAVES = 2 * NUM_SMS * ROWS + 17          # more than two waves at one CTA per SM
FWD_TOL = 2e-5                             # forward values, on the row's scale
BWD_TOL = 1e-4                             # dL/dy, dGates, dh0, on the row's scale
GRAD_L2, GRAD_MAX = 1e-4, 1e-3             # parameter gradients (grad_close)


def _cpu(x):
    return x.detach().cpu().double()


class Checks:
    """Collects (error, bound) per quantity, records them, then asserts every bound."""

    def __init__(self, what):
        self.what, self.errs = what, {}

    def rows(self, name, got, want, scale, tol):
        """max over each row of |got - want| / its scale; `scale` broadcasts over the rows'
        leading dimensions (the last dimension of got / want is the row)."""
        g, w = _cpu(got), want.detach().double()
        assert torch.isfinite(g).all(), (self.what, name, "unwritten or non-finite elements",
                                         torch.nonzero(~torch.isfinite(g))[:8].tolist())
        err = (g - w).abs().amax(-1) / (scale + 1e-30)
        self.add(name, float(err.max()) if err.numel() else 0.0, tol)

    def add(self, name, err, tol):
        self.errs[name] = (err, tol)

    def grads(self, got, want, names):
        for i, (g, w) in enumerate(zip(got, want)):
            assert torch.isfinite(g).all(), (self.what, names[i], "non-finite gradient")
            a, b = _cpu(g).reshape(-1), w.detach().double().reshape(-1)
            l2 = float((a - b).norm() / (b.norm() + 1e-30))
            mx = float((a - b).abs().max() / (b.abs().max() + 1e-30))
            self.add(f"grad.{names[i]}.l2", l2, GRAD_L2)
            self.add(f"grad.{names[i]}.max", mx, GRAD_MAX)

    def finish(self, test, **kv):
        _record(test, case=self.what, worst={k: e for k, (e, _) in self.errs.items()}, **kv)
        bad = {k: (e, t) for k, (e, t) in self.errs.items() if not e < t}
        assert not bad, (self.what, bad)


def _fwd_env(P, x, hs, layers, init=None):
    """[T, B]: per step and row, the largest |x||W_ih| + |b_ih| + |h_{t-1}||W_hh| + |b_hh| of
    any gate pre-activation at this step or an earlier one, in any layer (and `init` [B], the
    scale of the initial state)."""
    hs = hs.detach()
    terms = []
    for l in range(layers):
        w_ih, w_hh, b_ih, b_hh = (p.detach().abs() for p in P[4 * l: 4 * l + 4])
        inp = (x if l == 0 else hs[l - 1, 1:]).abs()
        terms.append((inp @ w_ih.T + b_ih + hs[l, :-1].abs() @ w_hh.T + b_hh).amax(-1))
    t = torch.stack(terms).amax(0)
    if init is not None:
        t = torch.maximum(t, init.unsqueeze(0))
    return t.cummax(0).values


def _bwd_env(per_step):
    """[T, B]: the largest of `per_step` [T, B] at this step or a later one."""
    return per_step.flip(0).cummax(0).values.flip(0)


def _fill_nan(*bufs):
    for b in bufs:
        b.fill_(NAN)


# ------------------------------------------------------------------------------------------
# MDN-RNN
# ------------------------------------------------------------------------------------------
class Mdn:
    def __init__(self, name, S, A, H, L, G, T, B, fit=False, div="state_dim", weights=(1, 1, 1)):
        self.name, self.S, self.A, self.H, self.L, self.G = name, S, A, H, L, G
        self.T, self.B, self.fit, self.div, self.weights = T, B, fit, div, weights
        self.NG, self.DX = (2 * S + 1) * G + 2, S + A

    def __repr__(self):
        return self.name


W = (0.7, 3.0, 0.4)  # next_state, not_terminal and reward loss weights: non-unit, unequal
MDN_CASES = [
    Mdn("H1_L1_G1_T1_B1", 3, 2, 1, 1, 1, 1, 1),
    Mdn("H3_L2_G31_DX3_B15_fit", 2, 1, 3, 2, 31, 2, 15, fit=True, weights=W),
    Mdn("H33_L4_G32_NG994_DX33_B17_div1", 15, 18, 33, 4, 32, 2, 17, div=None, weights=W),
    Mdn("H64_NG256_B16", 63, 1, 64, 2, 2, 2, 16),
    Mdn("H65_NG257_L1_B16_fit", 127, 2, 65, 1, 1, 2, 16, fit=True),
    Mdn("H127_DX2_L2_B17", 1, 1, 127, 2, 5, 2, 17, weights=W),
    Mdn("smem_H128_L4_NG1024_DX256_B17", 255, 1, 128, 4, 2, 2, 17, weights=W),
    Mdn("smem_H128_L4_G32_DX256_B15_fit_div1", 15, 241, 128, 4, 32, 2, 15, fit=True, div=None),
    Mdn("T64_H33_L2_B5", 4, 2, 33, 2, 3, 64, 5, weights=W),
    Mdn("T64_H65_L1_B3_fit_div1", 3, 3, 65, 1, 4, 64, 3, fit=True, div=None),
    Mdn("waves_B4241_H33_L2", 5, 2, 33, 2, 5, 2, B_WAVES, weights=W),
]


def _mdn_setup(case, seed):
    torch.manual_seed(seed)
    net = MemoryNetwork(case.S, case.A, case.H, case.L, case.G)
    with torch.no_grad():
        for p in net.mdnrnn.parameters():
            p.mul_(1.5)
    P64 = [p.detach().double().clone().requires_grad_(True) for p in net.mdnrnn.parameters()]
    w0, w1, w2 = case.weights
    tr = MDNRNNTrainer(net.cuda(), MDNRNNTrainerParameters(
        hidden_size=case.H, num_hidden_layers=case.L, num_gaussians=case.G, action_dim=case.A,
        next_state_loss_weight=w0, not_terminal_loss_weight=w1, reward_loss_weight=w2,
        fit_only_one_next_step=case.fit))
    g = torch.Generator().manual_seed(seed + 1)
    T, B, S, A = case.T, case.B, case.S, case.A
    b = dict(state=torch.randn(T, B, S, generator=g),
             action=torch.rand(T, B, A, generator=g) * 2 - 1,
             next_state=torch.randn(T, B, S, generator=g), reward=torch.randn(T, B, generator=g),
             not_terminal=(torch.rand(T, B, generator=g) > 0.2).float())
    batch = rlt.MemoryNetworkInput(
        state=rlt.FeatureData(b["state"].cuda()), next_state=rlt.FeatureData(b["next_state"].cuda()),
        action=rlt.FeatureData(b["action"].cuda()), reward=b["reward"].cuda(),
        not_terminal=b["not_terminal"].cuda(), time_diff=None, step=None)
    return tr, P64, b, batch


def _mdn_step(tr, case, batch):
    """One training step (forward, backward, wgrad) into NaN-filled buffers."""
    ws = tr._ws
    _fill_nan(ws.out, ws.hs, ws.cs, ws.xin, ws.acts, ws.dgates, ws.dy, ws.loss, ws.loss_partials,
              tr.memory_network.mdnrnn.arena.gpart)
    loss = tr._step(batch, case.S if case.div == "state_dim" else None, train=True)
    torch.cuda.synchronize()
    return loss


def _mdn_oracle(case, P64, b):
    b64 = {k: v.double() for k, v in b.items()}
    L, G, S = case.L, case.G, case.S
    out = LO.mdnrnn(P64, b64["state"], b64["action"], L, G)
    y = out["y"]
    w0, w1, w2 = case.weights
    ls = mo.losses(out, b64["next_state"], b64["reward"], b64["not_terminal"],
                   next_state_weight=w0, not_terminal_weight=w1, reward_weight=w2,
                   fit_only_one_next_step=case.fit,
                   state_dim=S if case.div == "state_dim" else None)
    # dL/dy of each loss; gy["loss"] is the kernels' dy
    gy = {k: torch.autograd.grad(ls[k], y, retain_graph=True)[0] for k in mo.LOSS_KEYS}
    ls["loss"].backward()
    return out, ls, gy


def _mdn_check(case, tr, P64, b, loss):
    ck = Checks(case.name)
    out, ls, gy = _mdn_oracle(case, P64, b)
    ws = tr._ws
    T, B, S, G, L, NG = case.T, case.B, case.S, case.G, case.L, case.NG
    GS = G * S
    x = out["x"].detach()
    # ---- exact ----
    assert torch.equal(ws.xin.cpu(), torch.cat([b["action"], b["state"]], -1)), "xin"
    zero = torch.zeros(L, B, case.H)
    assert torch.equal(ws.hs[:, 0].cpu(), zero) and torch.equal(ws.cs[:, 0].cpu(), zero), "slot 0"
    dy = _cpu(ws.dy)
    assert torch.isfinite(dy).all(), "dy unwritten"
    if case.fit:
        assert torch.equal(dy[:-1], torch.zeros_like(dy[:-1])), "dy before the last step"
    # ---- forward ----
    env = _fwd_env(P64, x, out["hs"], L)                                     # [T, B]
    ck.rows("hs", ws.hs[:, 1:], out["hs"][:, 1:], env, FWD_TOL)
    ck.rows("cs", ws.cs[:, 1:], out["cs"][:, 1:], env, FWD_TOL)
    ck.rows("acts", ws.acts, out["acts"], env, FWD_TOL)
    wg, bg = P64[4 * L].detach(), P64[4 * L + 1].detach()
    top = out["top"].detach()
    head = (top.abs() @ wg.abs().T + bg.abs()).amax(-1) + env * float(wg.abs().sum(1).max())
    y = out["y"].detach()
    o = _cpu(ws.out)
    ck.rows("out.mus", o[..., :GS], y[..., :GS], head, FWD_TOL)
    # sigma = exp(y): its relative error is the absolute error of y
    sig_k, sig_r = o[..., GS:2 * GS], torch.exp(y[..., GS:2 * GS])
    ck.rows("out.sigmas", sig_k / sig_r, torch.ones_like(sig_r), head, FWD_TOL)
    ck.rows("out.logpi", o[..., 2 * GS:2 * GS + G], out["logpi"], 2 * head, FWD_TOL)
    ck.rows("out.reward", o[..., NG - 2:NG - 1], y[..., NG - 2:NG - 1], head, FWD_TOL)
    ck.rows("out.not_terminal", o[..., NG - 1:], y[..., NG - 1:], head, FWD_TOL)
    # each loss against the first-order spread of its terms' errors
    lk = _cpu(loss)
    for i, k in enumerate(mo.LOSS_KEYS):
        r = float(ls[k].detach())
        scale = float((gy[k].abs() * head.unsqueeze(-1)).sum()) + abs(r)
        ck.add(f"loss.{k}", abs(float(lk[i]) - r) / scale, FWD_TOL)
    # ---- backward ----
    dy_r = gy["loss"]
    in_loss = slice(T - 1, T) if case.fit else slice(0, T)
    dy_scale = dy_r.abs().amax(-1) * torch.clamp(head, min=1.0)
    ck.rows("dy", dy[in_loss], dy_r[in_loss], dy_scale[in_loss], BWD_TOL)
    dg_r = LO.dgates(out)
    per_step = torch.maximum((dy_r.abs() @ wg.abs()).amax(-1), dg_r.abs().amax(-1).amax(0))
    ck.rows("dgates", ws.dgates, dg_r, _bwd_env(per_step), BWD_TOL)
    names = [f"l{l}.{n}" for l in range(L) for n in ("w_ih", "w_hh", "b_ih", "b_hh")]
    ck.grads(tr.mdnrnn_grads(), [p.grad for p in P64], names + ["gmm.w", "gmm.b"])
    return ck


@pytest.mark.parametrize("case", MDN_CASES, ids=repr)
def test_mdnrnn_train_step_matches_fp64(case):
    tr, P64, b, batch = _mdn_setup(case, seed=case.H + case.G + case.T)
    tr._step(batch, None, train=True)  # allocates tr._ws and the gradient partials
    loss = _mdn_step(tr, case, batch)
    _mdn_check(case, tr, P64, b, loss).finish("lstm_edges_mdnrnn", T=case.T, B=case.B)


def test_mdnrnn_two_launches_are_bit_identical_over_two_waves():
    case = MDN_CASES[-1]
    assert case.B == B_WAVES and -(-case.B // ROWS) > 2 * NUM_SMS
    tr, _, _, batch = _mdn_setup(case, seed=3)
    tr._step(batch, None, train=True)
    runs = []
    for _ in range(2):
        loss = _mdn_step(tr, case, batch).clone()
        assert int(tr._ws.counter.item()) == 0
        runs.append((loss, [g.clone() for g in tr.mdnrnn_grads()]))
    assert torch.isfinite(runs[0][0]).all()
    assert torch.equal(runs[0][0], runs[1][0])
    for g0, g1 in zip(runs[0][1], runs[1][1]):
        assert torch.isfinite(g0).all() and torch.equal(g0, g1)


# ------------------------------------------------------------------------------------------
# Seq2Reward
# ------------------------------------------------------------------------------------------
class S2r:
    def __init__(self, name, S, A, H, L, T, B, gamma=0.9):
        self.name, self.S, self.A, self.H, self.L, self.T, self.B = name, S, A, H, L, T, B
        self.gamma = gamma

    def __repr__(self):
        return self.name


S2R_CASES = [
    S2r("H1_L1_A1_B17", 3, 1, 1, 1, 5, 17),
    S2r("H33_L4_A16_B15", 5, 16, 33, 4, 3, 15, gamma=1.0),
    S2r("H65_L1_A3_B16", 7, 3, 65, 1, 4, 16),
    S2r("H128_L4_A4_B17", 20, 4, 128, 4, 3, 17, gamma=0.5),
    S2r("T64_valid_1_to_64_H33_L2_B64", 3, 2, 33, 2, 64, 64),
    S2r("waves_B4241_H33_L2", 4, 2, 33, 2, 2, B_WAVES),
]


def _s2r_setup(case, seed):
    torch.manual_seed(seed)
    net = Seq2RewardNetwork(case.S, case.A, case.H, case.L)
    with torch.no_grad():
        for p in net.parameters():
            p.mul_(1.5)
    P64 = [p.detach().double().clone().requires_grad_(True) for p in net.parameters()]
    g = torch.Generator().manual_seed(seed + 1)
    T, B = case.T, case.B
    b = dict(state=torch.randn(1, B, case.S, generator=g),
             action=F.one_hot(torch.randint(case.A, (T, B), generator=g), case.A).float(),
             reward=torch.randn(T, B, generator=g),
             valid=torch.arange(B) % T + 1)  # every valid step 1 .. T
    b["valid"] = b["valid"][torch.randperm(B, generator=g)]
    return net.cuda(), P64, b


def _s2r_run(net, b, gamma, ws=None):
    """Training forward, backward and wgrad into NaN-filled buffers (`ws` from an earlier
    call; None allocates)."""
    st, act = b["state"].cuda(), b["action"].cuda()
    valid, reward = b["valid"].cuda(), b["reward"].cuda()
    if ws is not None:
        _fill_nan(ws.acc_reward, ws.target, ws.hs, ws.cs, ws.acts, ws.dgates, ws.dy, ws.dh0,
                  ws.loss, ws.loss_partials, net.arena.gpart)
    ws = s2r_forward(net, st, act, valid, ws, reward=reward, gamma=gamma, train=True)
    splits = _lib.lib().rb200_wgrad_splits(act.shape[0] * act.shape[1])
    backward_wgrad(net, ws, splits, ensure_gpart(net.arena, splits))
    torch.cuda.synchronize()
    return ws


def _s2r_check(case, net, ws, P64, b):
    ck = Checks(case.name)
    T, B, L, H = case.T, case.B, case.L, case.H
    s0 = b["state"][0].double()
    act = b["action"].double()
    v = b["valid"]
    out = LO.seq2reward(P64, s0, act, L, v)
    acc = out["acc_reward"]
    acc.retain_grad()
    tg = so.target(b["reward"], v, case.gamma)
    loss = F.mse_loss(acc, tg.double())
    loss.backward()
    # ---- exact ----
    hs0 = ws.hs[:, 0].cpu()
    for l in range(1, L):
        assert torch.equal(hs0[l], hs0[0]), ("h0 differs between layers", l)
    assert torch.equal(ws.cs[:, 0].cpu(), torch.zeros(L, B, H)), "c0"
    assert torch.equal(ws.target.cpu(), tg.squeeze(1).float()), "target"
    dy = _cpu(ws.dy)
    dg = _cpu(ws.dgates)
    assert torch.isfinite(dy).all() and torch.isfinite(dg).all()
    t_idx = torch.arange(T).unsqueeze(1)
    off = t_idx != (v - 1).unsqueeze(0)                                    # [T, B]
    assert torch.equal(dy[off], torch.zeros(int(off.sum()), dtype=torch.float64)), "dy off step"
    after = t_idx >= v.unsqueeze(0)
    assert torch.equal(dg[:, after], torch.zeros_like(dg[:, after])), "dgates after valid_step"
    # ---- forward ----
    w_map, b_map = P64[4 * L + 2].detach(), P64[4 * L + 3].detach()
    init = (s0.abs() @ w_map.abs().T + b_map.abs()).amax(-1)
    env = _fwd_env(P64, act, out["hs"], L, init)
    ck.rows("hs0", ws.hs[:, 0], out["hs"][:, 0], init, FWD_TOL)
    ck.rows("hs", ws.hs[:, 1:], out["hs"][:, 1:], env, FWD_TOL)
    ck.rows("cs", ws.cs[:, 1:], out["cs"][:, 1:], env, FWD_TOL)
    ck.rows("acts", ws.acts, out["acts"], env, FWD_TOL)
    w_lin, b_lin = P64[4 * L].detach(), P64[4 * L + 1].detach()
    sel = out["top"].detach()[v - 1, torch.arange(B)]
    head = ((sel.abs() @ w_lin.abs().T + b_lin.abs()).reshape(-1)
            + env[v - 1, torch.arange(B)] * float(w_lin.abs().sum()))
    ck.rows("acc_reward", ws.acc_reward, acc, head, FWD_TOL)
    g_acc = acc.grad.reshape(-1)
    scale = float((g_acc.abs() * head).sum()) + float(loss)
    ck.add("loss", abs(float(ws.loss) - float(loss)) / scale, FWD_TOL)
    # ---- backward ----
    dy_r = torch.zeros(T, B, dtype=torch.float64)
    dy_r[v - 1, torch.arange(B)] = g_acc
    dy_scale = 2.0 / B * (head + tg.reshape(-1).abs())
    ck.rows("dy", dy.unsqueeze(-1), dy_r.unsqueeze(-1), dy_scale.unsqueeze(0), BWD_TOL)
    dg_r = LO.dgates(out)
    per_step = torch.maximum(dy_r.abs() * float(w_lin.abs().max()),
                             dg_r.abs().amax(-1).amax(0))
    benv = _bwd_env(per_step)
    ck.rows("dgates", ws.dgates, dg_r, benv, BWD_TOL)
    w_hh_sum = sum(float(P64[4 * l + 1].detach().abs().sum(0).max()) for l in range(L))
    ck.rows("dh0", ws.dh0, out["h0"].grad, benv[0] * w_hh_sum, BWD_TOL)
    names = ([f"l{l}.{n}" for l in range(L) for n in ("w_ih", "w_hh", "b_ih", "b_hh")]
             + ["lin.w", "lin.b", "map.w", "map.b"])
    ck.grads(param_grads(net.arena, list(net.parameters())), [p.grad for p in P64], names)
    return ck


@pytest.mark.parametrize("case", S2R_CASES, ids=repr)
def test_seq2reward_train_step_matches_fp64(case):
    net, P64, b = _s2r_setup(case, seed=case.H + case.A + case.T)
    ws = _s2r_run(net, b, case.gamma)
    ws = _s2r_run(net, b, case.gamma, ws)
    _s2r_check(case, net, ws, P64, b).finish("lstm_edges_seq2reward", T=case.T, B=case.B)


def test_seq2reward_rows_do_not_depend_on_their_cta():
    """Permuting the batch permutes acc_reward and every h bit for bit, at H 65 (three k
    chunks of W_hh): the forward runs without the k-chunk rotation, which the plan's
    bit-identity with the forward depends on."""
    case = S2r("perm_H65_L2", 5, 3, 65, 2, 6, 50)
    net, _, b = _s2r_setup(case, seed=11)
    ws = _s2r_run(net, b, case.gamma)
    acc, hs = ws.acc_reward.clone(), ws.hs.clone()
    perm = torch.randperm(case.B, generator=torch.Generator().manual_seed(2))
    bp = dict(state=b["state"][:, perm], action=b["action"][:, perm], reward=b["reward"][:, perm],
              valid=b["valid"][perm])
    ws = _s2r_run(net, bp, case.gamma, ws)
    assert torch.isfinite(acc).all()
    assert torch.equal(ws.acc_reward, acc[perm.cuda()])
    assert torch.equal(ws.hs, hs[:, :, perm.cuda()])


# ------------------------------------------------------------------------------------------
# world-model evaluators: every variant is mdn_step's copy of the forward, bit for bit
# ------------------------------------------------------------------------------------------
def _materialise(batch, c0, c1, value, A):
    """The batch with columns [c0, c1) of x = cat(action, state) set to `value` everywhere."""
    x = torch.cat([batch.action.float_features, batch.state.float_features], dim=-1).clone()
    x[:, :, c0:c1] = value.to(x.device)
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(x[:, :, A:].contiguous()), next_state=batch.next_state,
        action=rlt.FeatureData(x[:, :, :A].contiguous()), reward=batch.reward,
        not_terminal=batch.not_terminal, time_diff=None, step=None)


EVAL_CASES = [
    # (case, action feature starts, state feature starts)
    (Mdn("smem_H128_L4_NG1024", 255, 1, 128, 4, 2, 2, 17, weights=W), [0],
     list(range(0, 255, 32))),
    (Mdn("smem_H128_L4_G32_A241", 15, 241, 128, 4, 32, 2, 15), [0, 100, 200], [0, 3, 4, 10]),
    (Mdn("H33_L4_G32_B49_fit", 15, 2, 33, 4, 32, 3, 3 * ROWS + 1, fit=True), [0, 1],
     list(range(15))),
]


@pytest.mark.parametrize("case,a_starts,s_starts", EVAL_CASES, ids=[c[0].name for c in EVAL_CASES])
def test_evaluator_variants_equal_get_loss_and_forward(case, a_starts, s_starts):
    tr, _, _, batch = _mdn_setup(case, seed=case.S + case.A)
    S, A = case.S, case.A
    imp = FeatureImportanceEvaluator(tr, False, len(s_starts), len(a_starts), a_starts, s_starts)
    imp.evaluate(batch)
    got = imp._bufs.loss.clone()
    rows, _, _ = imp.variants(A, S)
    fill = imp.fill_values().cpu()
    assert len(rows) == 1 + len(a_starts) + len(s_starts)
    for v, (c0, c1, off) in enumerate(rows):
        ls = tr.get_loss(_materialise(batch, c0, c1, fill[off:off + c1 - c0], A), state_dim=S)
        want = torch.stack([ls[k] for k in ("gmm", "bce", "mse", "loss")])
        assert torch.isfinite(want).all()
        assert torch.equal(got[v], want), (v, got[v], want)
    perm = torch.randperm(case.B, generator=torch.Generator().manual_seed(4))
    sens = FeatureSensitivityEvaluator(tr, len(s_starts), s_starts)
    sens.evaluate(batch, perm=perm)
    mus = sens.means()
    with torch.no_grad():
        m0 = tr.memory_network(batch.state, batch.action).mus.clone()
        m1 = tr.memory_network(batch.state, rlt.FeatureData(
            batch.action.float_features[:, perm.cuda(), :])).mus.clone()
    assert torch.isfinite(m0).all()
    assert torch.equal(mus[0], m0)
    assert torch.equal(mus[1], m1)
