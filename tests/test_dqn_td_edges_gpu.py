"""The fused DQN TD step (K2) on both of its kernels -- dqn_td_tc_kernel (wgmma,
csrc/rb200_dqn_tc.cu) and dqn_td_rows_kernel in every forced row-tile instance
(csrc/rb200_dqn.cu) -- against float64, out to the shape limits of the wgmma plan and one step
past them.

* The trainer builds the arguments and the workspace (DQNTrainer._td_step), then every kernel
  is relaunched from `_last_td_call` into buffers prefilled with NaN (next_idx with -1), so a
  row a kernel never wrote cannot pass.
* The oracle is oracle/td_oracle (and per_oracle for importance weights) in float64.  It takes
  the kernel's fp32 decisions where fp32 noise decides them: the arg max where the top two
  masked values are within noise (all-masked rows: every action ties at -1e9 in fp32, so index
  0), the ReLU side of a unit within noise of 0 and the Huber branch of |d| within noise of 1.
  Those rows are counted, bounded and left out of the dZ comparison.
* Every row is compared on the scale of its own terms, with tolerances from _tol(K) for the
  contraction lengths K the row went through.
The case matrix covers the plan's paths: the register and the streamed input (S <= 128 and
above), a fourth 128-feature tile, A over 128, L = 1 and L = 8, short last k chunks, forward
only, importance weights, the POW discount and reward boosts.  Measured errors are appended to
$RB200_TEST_RECORD_DIR/test_measurements.jsonl when that directory exists."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import per_oracle as P
from oracle import td_oracle as O
from reagent_b200 import _lib
from tests.builders import _build_trainer, _record, _rlt_batch
from tests.kernel_util import (CFGS, E_SMEM, NAN, NUM_SMS, _cfg_id, _k2_image_bytes, _k2_tc_bytes,
                               _padded, _pick, _r8, _set_cfg, _tol)

pytestmark = pytest.mark.gpu

# rows within fp32 noise of a decision (ReLU kink, Huber corner, arg max) that float64 takes the
# other way, per launch: this many plus one per 256 rows
MAX_KNIFE_EDGE_ROWS = 2
GAMMA = 0.9


class Case:
    def __init__(self, name, S, sizes, A, B, acts=None, loss="huber", double_q=True, maxq=True,
                 weights=False, time_diff=False, boost=False, fwd_only=False, misaligned=False,
                 all_masked=False):
        self.name, self.S, self.sizes, self.A, self.B = name, S, list(sizes), A, B
        self.acts = list(acts) if acts is not None else ["relu"] * len(sizes)
        self.loss, self.double_q, self.maxq = loss, double_q, maxq
        self.weights, self.time_diff, self.boost = weights, time_diff, boost
        self.fwd_only, self.misaligned, self.all_masked = fwd_only, misaligned, all_masked

    def __repr__(self):
        return self.name

    @property
    def dims(self):
        return [self.S] + self.sizes + [self.A]

    def on_wgmma(self):
        return _k2_tc_bytes(self.dims, int(self.double_q), int(not self.fwd_only)) > 0

    def fwd_tol(self):
        """A forward chain: the contraction lengths of its layers add up."""
        return _tol(sum(self.dims))

    def bwd_tol(self):
        """dZ: the forward chain, then the transposed products back down."""
        return _tol(sum(self.dims) + sum(self.dims[1:]))


W4 = 2 * NUM_SMS * 32 + 1  # one row more than two waves of 32-row CTAs
CASES = [
    Case("S1_A2", 1, [8], 2, 33, all_masked=True),
    Case("S3_w9_mse_single", 3, [9], 9, 31, acts=["tanh"], loss="mse", double_q=False),
    Case("S4_w64_A1", 4, [64], 1, 32, time_diff=True),
    Case("S33_w65_129_B1", 33, [65, 129], 16, 1, acts=["relu", "leaky_relu"], weights=True),
    Case("S128_w128", 128, [128], 16, 4096, boost=True),                 # last register-path S
    Case("A128_boost", 9, [16], 128, 33, boost=True),
    Case("S129_streamed", 129, [64], 9, 33, loss="mse"),                  # scalar loads
    Case("S132_streamed", 132, [300], 9, 257),                            # vector loads
    Case("S132_misaligned", 132, [65], 9, 33, misaligned=True),
    Case("S192_config2", 192, [256, 128], 16, 4096, time_diff=True),     # inside the S edge
    Case("S480_streamed", 480, [8], 4, 33, loss="mse", weights=True),     # inside the S edge
    Case("w129_last_tile_1_row", 20, [129], 16, 65, acts=["sigmoid"]),
    Case("w385_fourth_tile", 8, [385], 8, 65, acts=["tanh"], double_q=False),
    Case("w472_inside", 8, [472], 8, 33),
    Case("A129_sarsa", 8, [8], 129, 64, maxq=False, loss="mse"),
    Case("A141_sarsa_weighted", 8, [8], 141, 33, maxq=False, weights=True),
    Case("A141_maxq_masked", 8, [8], 141, 33, all_masked=True, boost=True),
    Case("L1", 16, [], 9, 33, all_masked=True, boost=True, time_diff=True),
    Case("L1_fwd_only", 7, [], 2, 31, fwd_only=True),
    Case("L8_weighted", 12, [16] * 7, 5, 4096, weights=True, loss="mse",
         acts=["relu", "tanh", "relu", "sigmoid", "leaky_relu", "relu", "relu"]),
    Case("L3_mixed", 10, [24, 40], 3, 100, acts=["tanh", "leaky_relu"], maxq=False),
    Case("L4_mixed", 36, [20, 33, 17], 9, 257, acts=["sigmoid", "relu", "tanh"], loss="mse"),
    Case("two_waves", 16, [64], 4, W4, double_q=False),
    Case("fwd_only_streamed", 129, [300], 9, 33, fwd_only=True),
    Case("fwd_only_L8", 12, [16] * 7, 5, 65, fwd_only=True, all_masked=True),
    # one step past each edge of the wgmma plan: the row-tile kernel only
    Case("w473_outside", 8, [473], 8, 33),
    Case("A142_outside", 8, [8], 142, 33, maxq=False),
    Case("S193_outside", 193, [256, 128], 16, 64),
    Case("S481_outside", 481, [8], 4, 33, weights=True),
]
OUTSIDE = [c for c in CASES if c.name.endswith("_outside")]


def _trainer_and_batch(case, seed):
    meta = dict(S=case.S, A=case.A, B=case.B, sizes=case.sizes, acts=case.acts, gamma=GAMMA,
                tau=0.1, loss=case.loss, maxq=case.maxq, multi_steps=None,
                time_diff=case.time_diff, double_q=case.double_q, lr=1e-3, n_updates=1,
                boost={str(i): 0.25 * ((i % 5) - 2) for i in range(case.A)} if case.boost else None)
    torch.manual_seed(seed)
    t = _build_trainer(meta)
    with torch.no_grad():
        for p_ in t.q_network.parameters():
            if p_.dim() == 1:
                p_.add_(0.1 * torch.randn_like(p_))
        for p_, q_ in zip(t.q_network_target.parameters(), t.q_network.parameters()):
            p_.copy_(q_ + 0.05 * torch.randn_like(q_))
    g = torch.Generator().manual_seed(seed)
    B, S, A = case.B, case.S, case.A
    act = torch.randint(A, (B,), generator=g)
    nact = torch.randint(A, (B,), generator=g)
    nt = (torch.rand(B, 1, generator=g) > 0.25).float()
    mask = (torch.rand(B, A, generator=g) > 0.3).float()
    mask[torch.arange(B), nact] = 1.0
    if case.all_masked:
        # every fifth row has no possible next action; most of them are terminal, as ReAgent
        # builds them, and every third of them is not
        rows = torch.arange(0, B, 5)
        mask[rows] = 0.0
        nt[rows] = (torch.arange(rows.numel()) % 3 == 2).float().reshape(-1, 1)
    b = dict(state=torch.randn(B, S, generator=g), next_state=torch.randn(B, S, generator=g),
             reward=torch.randn(B, 1, generator=g),
             time_diff=(torch.tensor([0.0, 1.0, 7.0])[torch.randint(3, (B,), generator=g)]
                        .reshape(B, 1) if case.time_diff else torch.ones(B, 1)),
             step=None, not_terminal=nt, action=F.one_hot(act, A).float(),
             # SARSA: terminal rows have no next action at all (every action masked)
             next_action=F.one_hot(nact, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=mask)
    w = None
    if case.weights:
        w = torch.rand(B, generator=g) * 2.0
        w[3::7] = 0.0
    batch = _rlt_batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    return t, b, w, batch


def _net64(module, acts):
    dnn = module.fc.dnn
    return {"W": [s[0].weight.detach().cpu().double() for s in dnn],
            "b": [s[0].bias.detach().cpu().double() for s in dnn], "act": list(acts) + ["linear"]}


def _terms(net, x):
    """Per layer and row, the largest sum of magnitudes |W||h| + |b| behind any of the
    layer's outputs: the scale the layer's fp32 products carry, whatever they cancel to."""
    out = []
    for W, bias, a in zip(net["W"], net["b"], net["act"]):
        out.append((x.abs() @ W.abs().T + bias.abs()).amax(1))
        x = O._ACT[a](F.linear(x, W, bias))
    return out


def _dact(h, a):
    """|act'| through the activation's output, as the kernels take it"""
    return {"relu": (h > 0).double(), "leaky_relu": torch.where(h > 0, 1.0, 0.01).double(),
            "tanh": (1 - h * h).abs(), "sigmoid": (h * (1 - h)).abs(),
            "linear": torch.ones_like(h)}[a]


class Oracle:
    """The float64 side of one case; `check` compares one launch against it."""

    def __init__(self, case, t, b, w):
        self.case = case
        self.q = _net64(t.q_network, case.acts)
        self.qt = _net64(t.q_network_target, case.acts)
        self.b = {k: (v.double() if v is not None else None) for k, v in b.items()}
        self.w = None if w is None else w.double()
        bb, B, A = self.b, case.B, case.A
        self.boost = (t.reward_boosts.detach().cpu().double().reshape(1, -1) if case.boost else None)
        self.disc_src = bb["time_diff"] if case.time_diff else None
        kw = dict(gamma=GAMMA, double_q=case.double_q, maxq=case.maxq, loss=case.loss,
                  discount_src=self.disc_src, reward_boost=self.boost)
        if self.w is None:
            self.loss_ref, self.aux = O.dqn_td_loss(self.q, self.qt, bb, **kw)
        else:
            self.loss_ref, self.aux = P.weighted_td_loss(self.q, self.qt, bb, self.w, **kw)
        qn, qnt = O.mlp(self.q, bb["next_state"]), O.mlp(self.qt, bb["next_state"])
        mask = bb["possible_next_actions_mask"] if case.maxq else bb["next_action"]
        pen = O.ACTION_NOT_POSSIBLE_VAL * (1 - mask)
        self.keys = (qn if case.double_q else qnt) + pen
        self.vals = qnt + pen
        self.qnt_scale = torch.maximum(_terms(self.q, bb["next_state"])[-1],
                                       _terms(self.qt, bb["next_state"])[-1])
        self.all_masked = mask.sum(1) == 0
        # every action ties at -1e9 in fp32 only while |q| < 32 (half an fp32 ulp at 1e9)
        if bool(self.all_masked.any()):
            assert float(torch.maximum(qn.abs(), qnt.abs())[self.all_masked].max()) < 32
        self.terms = _terms(self.q, bb["state"])
        self.reward = bb["reward"].reshape(-1)
        if self.boost is not None:
            self.reward = self.reward + (bb["action"] * self.boost).sum(1)
        # gamma ** time_diff in fp32, as dqn_td_loss (and the kernels' powf) takes it
        self.disc = (torch.pow(GAMMA, self.disc_src.reshape(-1).float()).double()
                     if self.disc_src is not None
                     else torch.full((B,), GAMMA, dtype=torch.float64))
        self.nt = bb["not_terminal"].reshape(-1)
        top = self.keys.topk(min(2, A), dim=1).values
        self.top = top[:, 0]
        self.gap = top[:, 0] - top[:, 1] if A > 1 else torch.full((B,), float("inf"), dtype=torch.float64)
        self.noise = 4 * case.fwd_tol() * torch.clamp(self.qnt_scale, min=1.0)
        # forward of the online network on state, pre-activations kept for autograd
        self.zs, self.hs = [], []
        x = bb["state"]
        for W, bias, a in zip(self.q["W"], self.q["b"], self.q["act"]):
            W, bias = W.clone().requires_grad_(True), bias.clone().requires_grad_(True)
            z = F.linear(x, W, bias)
            z.retain_grad()
            x = O._ACT[a](z)
            self.zs.append(z)
            self.hs.append(x)
        assert torch.equal(self.hs[-1].detach(), self.aux["all_q"])
        self.q_sel = (self.hs[-1] * bb["action"]).sum(1)
        # d q_sel / d z_l row by row: dZ_l = g * J_l with g the loss's d / d q_sel
        self.J = [z_g.detach().clone() for z_g in torch.autograd.grad(self.q_sel.sum(), self.zs,
                                                                       retain_graph=True)]
        # the same chain on magnitudes, |W|^T |J| |act'|: the scale of the terms of each dZ
        L = len(self.zs)
        self.Jt = [None] * L
        self.Jt[-1] = self.J[-1].abs()
        for l in range(L - 2, -1, -1):
            self.Jt[l] = (self.Jt[l + 1] @ self.q["W"][l + 1].abs()) * _dact(self.hs[l].detach(), self.q["act"][l])

    def check(self, ws, what):
        """Compare one launch's outputs (in `ws`) with float64; returns (worst errors, knife rows)."""
        case, B, A = self.case, self.case.B, self.case.A
        worst = {}
        cpu = lambda x: x.detach().cpu().double()

        def rows(name, got, want, scale, tol, keep=None):
            g_, w_ = cpu(got).reshape(B, -1), want.detach().double().reshape(B, -1)
            assert torch.isfinite(g_).all(), (what, name, "unwritten rows",
                                              torch.nonzero(~torch.isfinite(g_).all(1)).reshape(-1)[:8])
            err = (g_ - w_).abs().amax(1) / (scale.reshape(-1) + 1e-30)
            if keep is not None:
                err = err[keep]
            e = float(err.max()) if err.numel() else 0.0
            assert e < tol, (what, name, "row", int(err.argmax()), e, tol)
            worst[name] = e

        # ---- arg max: exact, except at ties within fp32 noise ----
        idx_k = ws["next_idx"].cpu().long()
        idx_ref = self.aux["next_idx"].reshape(-1)
        knife_arg = (self.gap <= self.noise) & ~self.all_masked
        assert (idx_k[self.all_masked] == 0).all(), (what, "all-masked rows take index 0")
        sure = ~knife_arg & ~self.all_masked
        assert torch.equal(idx_k[sure], idx_ref[sure]), (what, "next_idx",
                                                         torch.nonzero(idx_k[sure] != idx_ref[sure])[:8])
        kk = torch.nonzero(knife_arg).reshape(-1)
        if kk.numel():
            picked = self.keys[kk, idx_k[kk]]
            assert (picked >= self.top[kk] - self.noise[kk]).all(), (what, "next_idx at a tie")
        idx = torch.where(knife_arg | self.all_masked, idx_k, idx_ref)
        next_q = self.vals.gather(1, idx.reshape(-1, 1)).reshape(-1)
        target = self.reward + self.disc * (next_q * self.nt)
        if not bool((knife_arg | self.all_masked).any()):
            assert torch.allclose(target, self.aux["target"].reshape(-1), rtol=0, atol=1e-12)

        fwd = case.fwd_tol()
        tgt_k = ws["td_target"].cpu()
        tgt_scale = self.reward.abs() + self.disc * self.nt * torch.maximum(next_q.abs(), self.qnt_scale)
        rows("td_target", tgt_k, target, tgt_scale, fwd)
        term = self.all_masked & (self.nt == 0)
        if bool(term.any()):
            # r + gamma * (-1e9 * 0): the reward (with its boost, added in fp32) bit for bit
            r32 = self.b["reward"].float().reshape(-1)
            if self.boost is not None:
                r32 = r32 + (self.b["action"].float() * self.boost.float()).sum(1)
            assert torch.equal(tgt_k[term], r32[term]), (what, "td_target of all-masked terminal rows")
        q_scale = self.terms[-1]
        rows("scores", ws["scores"], self.aux["all_q"], q_scale, fwd)
        rows("q_selected", ws["q_sel"], self.q_sel, q_scale, fwd)

        # ---- loss and dZ, autograd on the target that follows the kernel's arg max ----
        d = self.q_sel - target
        per_row = d * d if case.loss == "mse" else F.smooth_l1_loss(self.q_sel, target, reduction="none")
        wv = self.w if self.w is not None else torch.ones(B, dtype=torch.float64)
        loss = torch.mean(wv * per_row)
        if not bool((knife_arg | self.all_masked).any()):
            assert abs(float(loss) - float(self.loss_ref)) <= 1e-12 * max(1.0, abs(float(loss)))
        lk = float(ws["loss"].cpu())
        e = abs(lk - float(loss)) / (float(torch.mean(wv * per_row.detach().abs())) + 1e-30)
        assert e < max(fwd, _tol(B)), (what, "loss", lk, float(loss), e)
        worst["loss"] = e

        L = len(self.zs)
        if case.fwd_only:
            # nothing of the backward workspace is touched
            for x in ws["net"].hidden + ws["net"].dz:
                assert torch.isnan(x).all(), (what, "forward-only launch wrote the gradient workspace")
            return worst, int(knife_arg.sum())
        dz64 = torch.autograd.grad(loss, self.zs, retain_graph=True)
        knife = knife_arg.clone()
        # Huber corner: |d| within noise of 1
        c = 2.0 if case.loss == "mse" else 1.0
        # d = q_sel - target carries the errors of both products behind it
        d_scale = q_scale + tgt_scale
        if case.loss == "huber":
            knife |= ((d.detach().abs() - 1).abs() <= 4 * fwd * d_scale)
        # ReLU / leaky-ReLU side of every hidden unit, from the saved activations
        for l in range(L - 1):
            h64 = self.hs[l].detach()
            hk = cpu(ws["net"].hidden[l])
            rows(f"hidden{l}", hk, h64, self.terms[l], _tol(sum(self.case.dims[:l + 2])))
            if self.q["act"][l] in ("relu", "leaky_relu"):
                knife |= ((hk > 0) != (h64 > 0)).any(1)
        n_knife = int(knife.sum())
        assert n_knife <= MAX_KNIFE_EDGE_ROWS + B // 256, (what, "knife-edge rows", n_knife)
        # dZ_l = g J_l: the error of g is that of d (a difference of q_sel and the target)
        g_abs = (dz64[-1].abs().amax(1) / (self.J[-1].abs().amax(1) + 1e-300))
        g_err = c * wv / B * d_scale
        keep = ~knife
        for l in range(L):
            scale = self.Jt[l].amax(1) * (g_abs + g_err)
            rows(f"dz{l}", ws["net"].dz[l], dz64[l], scale, case.bwd_tol(), keep=keep)
        return worst, n_knife


def _fill_nan(ws):
    for k in ("scores", "td_target", "q_sel", "loss"):
        ws[k].fill_(NAN)
    for x in ws["net"].hidden + ws["net"].dz:
        x.fill_(NAN)
    ws["next_idx"].fill_(-1)


def _prepare(case, seed):
    t, b, w, batch = _trainer_and_batch(case, seed)
    if case.fwd_only:
        t.compute_td_loss_only(batch)
    else:
        t._td_step(batch, sample_weight=None if w is None else w.cuda())
    torch.cuda.synchronize()
    call = t._last_td_call
    assert (call[-1] is not None) == case.on_wgmma(), (case, "K2 ran on the wrong kernel")
    assert int(call[2].do_backward) == int(not case.fwd_only)
    assert (int(call[2].sample_weight or 0) != 0) == case.weights
    keep = []
    if case.misaligned:
        xs = _padded((case.B, case.S), offset=1)
        xs.copy_(b["state"])
        assert xs.data_ptr() % 16 != 0
        call[2].state = xs.data_ptr()
        keep.append(xs)
    return t, b, w, keep


def _run_rows(t, cfg, monkeypatch):
    qd, qtd, a, wsc, _, _ = t._last_td_call
    _set_cfg(monkeypatch, cfg)
    _fill_nan(t._ws)
    rc = _lib.lib().rb200_dqn_td_step(qd, qtd, a, wsc, _lib.cur_stream())
    torch.cuda.synchronize()
    _set_cfg(monkeypatch, None)
    return rc


def _run_tc(t, pack):
    qd, qtd, a, wsc, _, _ = t._last_td_call
    _fill_nan(t._ws)
    rc = _lib.lib().rb200_dqn_td_step_tc(qd, qtd, a, wsc, pack.data_ptr(), pack.numel(), 0,
                                         _lib.cur_stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("case", CASES, ids=repr)
def test_k2_kernels_match_fp64(case, monkeypatch):
    t, b, w, keep = _prepare(case, seed=case.B + case.S + case.A)
    ref = Oracle(case, t, b, w)
    pack = t._last_td_call[-1]
    results = {}
    if pack is not None:
        assert _run_tc(t, pack) == 0
        results["wgmma"] = ref.check(t._ws, f"{case}/wgmma")
    hmax = max(case.sizes) if case.sizes else 0
    extra = 3 * (((case.A + 3) & ~3) + 4) + 2
    for cfg in CFGS:
        fits = _pick(cfg, case.B, case.S, hmax, 1, 3, extra) is not None
        rc = _run_rows(t, cfg, monkeypatch)
        if not fits:
            assert rc == E_SMEM, (case, _cfg_id(cfg), rc)
            continue
        assert rc == 0, (case, _cfg_id(cfg), rc, _lib.lib().rb200_last_error())
        results[f"rows_{_cfg_id(cfg)}"] = ref.check(t._ws, f"{case}/rows_{_cfg_id(cfg)}")
    assert results
    for k, (worst, knife) in results.items():
        _record("k2_edges", case=case.name, kernel=k, B=case.B, knife_edge_rows=knife, worst=worst)


@pytest.mark.parametrize("case", OUTSIDE, ids=repr)
def test_wgmma_entry_refuses_shapes_past_its_plan(case):
    """One step past the plan the trainer holds no pack (the rows kernel ran, checked against
    float64 above) and a direct call returns RB200_E_SMEM without launching anything."""
    t, b, w, keep = _prepare(case, seed=1)
    qd, qtd, a, wsc, _, pack = t._last_td_call
    assert pack is None
    scratch = torch.zeros(8 << 20, dtype=torch.uint8, device="cuda")
    for packed in (0, 1):
        _fill_nan(t._ws)
        torch.cuda.synchronize()
        rc = _lib.lib().rb200_dqn_td_step_tc(qd, qtd, a, wsc, scratch.data_ptr(), scratch.numel(),
                                             packed, _lib.cur_stream())
        torch.cuda.synchronize()
        assert rc == E_SMEM, (case, packed, rc)
        assert torch.isnan(t._ws["loss"]).all() and torch.isnan(t._ws["scores"]).all()
        assert (t._ws["next_idx"] == -1).all()
    assert int(scratch.count_nonzero()) == 0


# ------------------------------------------------------------------------------------------
# weight images
# ------------------------------------------------------------------------------------------
def _image(Wnp, transpose):
    """The documented image of A = W (or W^T): per (128-row tile t, 32-k chunk c) a block
    [k/4][rows][4] with quad stride rows8 * 16 + 16 bytes; returns {float offset: value} over
    every position a chunk defines (rows < rows8, k < kl8), zeros past N and K."""
    A = Wnp.T if transpose else Wnp
    N, K = A.shape
    offs, vals = [], []
    for t in range((N + 127) // 128):
        rows8 = _r8(min(N - 128 * t, 128))
        lbo4 = rows8 * 4 + 4
        for c in range((K + 31) // 32):
            kl8 = _r8(min(K - 32 * c, 32))
            base = t * (_r8(K) // 4) * (128 * 4 + 4) + c * 8 * lbo4
            r, k = np.meshgrid(np.arange(rows8), np.arange(kl8), indexing="ij")
            offs.append((base + (k >> 2) * lbo4 + r * 4 + (k & 3)).reshape(-1))
            m, kg = 128 * t + r, 32 * c + k
            v = np.zeros(r.shape, np.float32)
            inside = (m < N) & (kg < K)
            v[inside] = A[m[inside], kg[inside]]
            vals.append(v.reshape(-1))
    return np.concatenate(offs), np.concatenate(vals)


@pytest.mark.parametrize("dims", [[1, 129, 7], [7, 400, 9], [33, 129, 1], [480, 8, 4],
                                  [8, 8, 141], [9, 385, 65, 9]], ids=str)
@pytest.mark.parametrize("do_backward", [0, 1])
def test_pack_kernel_writes_the_documented_image_layout(dims, do_backward):
    from reagent_b200.models import FullyConnectedDQN

    assert _k2_tc_bytes(dims, 1, do_backward) > 0
    torch.manual_seed(len(dims) + dims[0])
    q = FullyConnectedDQN(dims[0], dims[-1], dims[1:-1], ["relu"] * (len(dims) - 2)).cuda()
    qt = q.get_target_network().cuda()
    with torch.no_grad():
        for p_ in list(q.parameters()) + list(qt.parameters()):
            p_.copy_(torch.randn_like(p_))
    nbytes = _k2_tc_bytes(dims, 1, do_backward)
    buf = torch.full((nbytes // 4,), NAN, device="cuda")
    rc = _lib.lib().rb200_dqn_tc_pack(q.arena.desc(), qt.arena.desc(), 1, do_backward,
                                      buf.data_ptr(), nbytes, _lib.cur_stream())
    _lib.check(rc, "rb200_dqn_tc_pack")
    torch.cuda.synchronize()
    got = buf.cpu().numpy().view(np.uint32)
    L = len(dims) - 1
    Ws = [s[0].weight.detach().cpu().numpy() for s in q.fc.dnn]
    Wt = [s[0].weight.detach().cpu().numpy() for s in qt.fc.dnn]
    jobs = [(W, 0) for W in Ws] + [(W, 0) for W in Wt]
    if do_backward:
        jobs += [(Ws[l], 1) for l in range(1, L)]
    off = 0
    for W, tr in jobs:
        N, K = (W.shape[1], W.shape[0]) if tr else W.shape
        o, v = _image(W, tr)
        assert np.array_equal(got[off // 4 + o], v.view(np.uint32)), (dims, tr, N, K)
        off += _k2_image_bytes(N, K)
    assert off + 4096 == nbytes


# ------------------------------------------------------------------------------------------
# the cached images of the two pack keys, and the loss reduction's counter
# ------------------------------------------------------------------------------------------
def test_td_loss_only_interleaved_with_train_batch_reads_current_weights():
    """compute_td_loss_only packs its forward-only images on every call and train_batch keeps
    the backward images written by the Adam step: interleaved for three updates, each loss must
    be that of the parameters at that moment (a stale image would give an earlier update's)."""
    case = Case("interleave", 33, [129], 9, 512)
    t, b, w, meta_batch = _trainer_and_batch(case, seed=5)
    _, b_eval, _, batch_eval = _trainer_and_batch(case, seed=6)
    qo = _net64(t.q_network, case.acts)
    qto = _net64(t.q_network_target, case.acts)
    qo = O.clone_net(qo, requires_grad=True)
    adam = O.AdamState(O.net_params(qo), lr=1e-3)
    b64 = {k: (v.double() if v is not None else None) for k, v in b.items()}
    e64 = {k: (v.double() if v is not None else None) for k, v in b_eval.items()}
    kw = dict(gamma=GAMMA, double_q=True, maxq=True, loss="huber")
    for it in range(3):
        ev = float(t.compute_td_loss_only(batch_eval))
        assert t._last_td_call[-1] is not None and int(t._last_td_call[2].do_backward) == 0
        now, now_t = _net64(t.q_network, case.acts), _net64(t.q_network_target, case.acts)
        want, _ = O.dqn_td_loss(now, now_t, e64, **kw)
        assert abs(ev - float(want)) <= case.fwd_tol() * max(1.0, abs(float(want))), (it, ev, float(want))
        lo, _, _ = O.dqn_update(qo, qto, adam, b64, tau=0.1, **kw)
        got = float(t.train_batch(meta_batch, it))
        assert t._last_td_call[-1] is not None and int(t._last_td_call[2].do_backward) == 1
        assert abs(got - lo) <= 2e-5 * max(1.0, abs(lo)), (it, got, lo)
        _record("k2_interleave", it=it, eval_loss=ev, eval_want=float(want), loss=got, loss_want=lo)


@pytest.mark.parametrize("path", ["wgmma", "rows"])
def test_k2_loss_is_bit_identical_across_launches_at_65536_rows(path, monkeypatch):
    """The loss is reduced over the CTAs in a fixed order by the last one to finish, which
    resets tile_counter: two launches give the same bits, and the counter is 0 after each."""
    case = Case("det", 128, [256, 128], 16, 65536)
    t, b, w, _ = _prepare(case, seed=7)
    pack = t._last_td_call[-1]
    assert pack is not None
    losses = []
    for _ in range(2):
        rc = _run_tc(t, pack) if path == "wgmma" else _run_rows(t, None, monkeypatch)
        assert rc == 0
        assert int(t._ws["counter"].item()) == 0
        losses.append(t._ws["loss"].clone())
    assert torch.isfinite(losses[0]).all()
    assert torch.equal(losses[0], losses[1]), [float(x) for x in losses]
