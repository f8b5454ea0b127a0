"""The fused SAC / TD3 row-tile kernels (csrc/rb200_actor_critic.cu) against the float64
restatement of oracle/ac_fp64.py, driven through the trainers' own launch helpers
(ActorCriticBase._critic_step / _actor_step, SACTrainer._value_step) in every row-tile
configuration (RB200_FORCE_CFG) and at the regimes where the kernels depart from a plain MLP.

* Every output and workspace buffer is prefilled with NaN, so a row the kernel never wrote
  cannot pass, and every row is compared on its own scale (the first and last row of the
  ragged last tile included).
* A forced tile that does not fit must be refused with RB200_E_SMEM, exactly when the mirror
  of pick_rows_cfg says so; a launch that succeeds therefore ran that instantiation.
* The oracle takes the kernel's fp32 decisions where fp32 noise decides them (the saved
  activations for the activation derivatives, the squashed actions, the log-prob clamp mask)
  and every one of those inputs is itself checked against float64.  How many decisions float64
  would have taken the other way is counted and bounded.

Random weights are scaled by 1/sqrt(fan_in), so every row is O(1).  Measured errors are
appended to $RB200_TEST_RECORD_DIR/test_measurements.jsonl when that directory exists."""
import math

import numpy as np
import pytest
import torch

from oracle import ac_fp64 as X
from reagent_b200 import _lib
from tests.builders import _pbatch, _record
from tests.kernel_util import CFGS, E_SMEM, NAN, TOL, _cfg_id, _pick, _set_cfg, _tol

pytestmark = pytest.mark.gpu

BATCHES = [1, 15, 16, 17, 31, 32, 33]
# at most this many rows may sit within fp32 noise of a decision (a ReLU kink, a clamp bound)
# that float64 takes the other way; the oracle follows the kernel's side on them
MAX_KNIFE_EDGE_ROWS = 2


def _net(dims, acts, g, bias=0.3):
    return {"W": [torch.randn(dims[i + 1], dims[i], generator=g) / math.sqrt(dims[i])
                  for i in range(len(acts))],
            "b": [torch.randn(dims[i + 1], generator=g) * bias for i in range(len(acts))],
            "act": list(acts)}


def _load(module, net):
    fc = module.fc if hasattr(module, "fc") else module
    with torch.no_grad():
        for i, seq in enumerate(fc.dnn):
            seq[0].weight.copy_(net["W"][i])
            seq[0].bias.copy_(net["b"][i])


class Case:
    """One network shape: S, A, hidden sizes and activations shared by actor and critics."""

    def __init__(self, S, A, sizes, acts, batches=(17, 33)):
        self.S, self.A, self.sizes, self.acts = S, A, list(sizes), list(acts)
        self.batches = list(batches)

    def __repr__(self):
        return f"S{self.S}A{self.A}{self.sizes}"

    def nets(self, algo, g, loc_bias=None, sl_bias=None, twin_tie=False, value=False,
             sl_weight_scale=None):
        S, A = self.S, self.A
        NO = 2 * A if algo == "sac" else A
        actor = _net([S] + self.sizes + [NO], self.acts + ["linear" if algo == "sac" else "tanh"], g)
        if loc_bias is not None:
            actor["b"][-1][:A] = torch.as_tensor(loc_bias, dtype=torch.float32)
        if sl_bias is not None:
            actor["b"][-1][A:] = torch.as_tensor(sl_bias, dtype=torch.float32)
        if sl_weight_scale is not None:
            actor["W"][-1][A:] *= sl_weight_scale
        q1 = _net([S + A] + self.sizes + [1], self.acts + ["linear"], g)
        q2 = q1 if twin_tie else _net([S + A] + self.sizes + [1], self.acts + ["linear"], g)
        v = _net([S] + self.sizes + [1], self.acts + ["linear"], g) if value else None
        return actor, q1, q2, v

    def hmax(self):
        return max(self.sizes)

    def chain(self):
        """Bound of a forward or dZ chain through a critic: the contraction lengths of its
        layers add up (measured on an H100: 1.4e-5 for a squashed action through the
        [256, 256, 256 -> 64] actor of bench config 4, 3.2e-5 for a log-prob through
        [700, 600 -> 12])."""
        return _tol(self.S + self.A + sum(self.sizes))


CASES = [
    Case(8, 3, [64, 32], ["relu", "tanh"], batches=BATCHES),
    Case(7, 3, [33], ["leaky_relu"]),                                   # S + A = 10
    Case(29, 6, [40, 24], ["relu", "relu"]),                            # a' straddles k = 32
    Case(5, 1, [16], ["tanh"]),                                         # A = 1
    Case(16, 64, [48], ["relu"]),                                       # A = 64
    Case(9, 4, [300], ["relu"]),                                        # hidden over 256
    Case(6, 2, [24, 257, 20], ["softplus", "relu", "sigmoid"]),         # 3 layers, mixed
    Case(700, 6, [600], ["relu"], batches=(17,)),                       # only k-chunk 16 fits
    Case(12, 5, [96, 64], ["relu", "leaky_relu"], batches=(2113, 4097)),  # 32-row default tile
]


# ------------------------------------------------------------------------------------------
# trainers and launches
# ------------------------------------------------------------------------------------------
def _sac(case, actor, q1, q2, value=None, *, gamma=0.9, alpha=0.2, learn_alpha=True,
         target_entropy=-2.0, backprop=True, crr=None, uniform_prior=True):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.training import CRRWeightFn, SACTrainer

    S, A = case.S, case.A
    am = GaussianFullyConnectedActor(S, A, case.sizes, case.acts)
    m1 = FullyConnectedCritic(S, A, case.sizes, case.acts)
    m2 = None if q2 is None else FullyConnectedCritic(S, A, case.sizes, case.acts)
    vm = None if value is None else FloatFeatureFullyConnected(S, 1, case.sizes, case.acts)
    for m, n in ((am, actor), (m1, q1), (m2, q2), (vm, value)):
        if m is not None:
            _load(m, n)
    kw = {} if learn_alpha else {"alpha_optimizer": None}
    t = SACTrainer(am, m1, m2, vm, rl=RLParameters(gamma=gamma, target_update_rate=0.1),
                   entropy_temperature=alpha, target_entropy=target_entropy,
                   backprop_through_log_prob=backprop, logged_action_uniform_prior=uniform_prior,
                   crr_config=None if crr is None else CRRWeightFn(**crr), **kw)
    return t.cuda()


def _td3(case, actor, q1, q2, *, gamma=0.9, noise_variance=0.2, noise_clip=0.5):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedActor, FullyConnectedCritic
    from reagent_b200.training import TD3Trainer

    S, A = case.S, case.A
    am = FullyConnectedActor(S, A, case.sizes, case.acts)
    m1 = FullyConnectedCritic(S, A, case.sizes, case.acts)
    m2 = None if q2 is None else FullyConnectedCritic(S, A, case.sizes, case.acts)
    for m, n in ((am, actor), (m1, q1), (m2, q2)):
        if m is not None:
            _load(m, n)
    t = TD3Trainer(am, m1, m2, rl=RLParameters(gamma=gamma, target_update_rate=0.1),
                   noise_variance=noise_variance, noise_clip=noise_clip)
    return t.cuda()


def _batch(case, B, g, reward_nan_row=None, terminal="mixed"):
    S, A = case.S, case.A
    b = {"state": torch.randn(B, S, generator=g), "next_state": torch.randn(B, S, generator=g),
         "action": torch.rand(B, A, generator=g) * 2 - 1,
         "next_action": torch.zeros(B, A), "reward": torch.randn(B, 1, generator=g)}
    if terminal == "all":
        b["not_terminal"] = torch.zeros(B, 1)
    else:
        b["not_terminal"] = (torch.rand(B, 1, generator=g) > 0.25).float()
    if reward_nan_row is not None:
        b["reward"][reward_nan_row] = NAN
    return b, _pbatch({k: v.cuda() for k, v in b.items()})


def _nan_ws(t, B):
    """Build (or reuse) the trainer's workspace for B rows and fill every buffer with NaN."""
    ws = t._workspace(B, torch.device("cuda", torch.cuda.current_device()))
    for k, v in ws.items():
        if isinstance(v, torch.Tensor) and v.is_floating_point():
            v.fill_(NAN)
        elif hasattr(v, "hidden"):
            for x in v.hidden + v.dz + ([v.input] if v.input is not None else []):
                x.fill_(NAN)
    return ws


def _inject(t, noise):
    t.noise_hook = lambda name, shape, device: noise[name].to(device)


def _extra_fill(base, B, A, want_min_q=False):
    """The trainer's filler plus next_action_out (and min_q_out) into NaN-filled buffers."""
    bufs = {"action": torch.full((B, A), NAN, device="cuda")}
    if want_min_q:
        bufs["min_q"] = torch.full((B,), NAN, device="cuda")

    def fill(a, pins):
        base(a, pins)
        a.next_action_out = bufs["action"].data_ptr()
        if want_min_q:
            a.min_q_out = bufs["min_q"].data_ptr()
    return fill, bufs


def _launch(fn):
    """(ok, error): a forced tile that does not fit raises with RB200_E_SMEM."""
    try:
        fn()
        torch.cuda.synchronize()
        return True, None
    except _lib.Rb200Error as e:
        return False, str(e)


def _tile_rows(cfg, B, din, hmax, extra):
    p = _pick(cfg, B, din, hmax, 1, 3, extra)
    return None if p is None else (p[0] // 64) * 4


def _critic_extra(NO):
    ld_o = ((max(NO, 8) + 3) & ~3) + 12
    return ld_o + 16 + 4


def _actor_extra(NO):
    ld_o = ((max(NO, 8) + 3) & ~3) + 12
    return 3 * ld_o + 16 + 4


# ------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------
class Cmp:
    """Row-by-row comparison of kernel outputs with float64, tracking the worst error per
    output name."""

    def __init__(self, B, R, what, skip_rows=None):
        self.B, self.R, self.what = B, R, what
        self.worst = {}
        self.keep = torch.ones(B, dtype=torch.bool)
        if skip_rows is not None:
            self.keep[skip_rows] = False

    def rows(self, name, got, want, tol=TOL):
        B = self.B
        g = torch.as_tensor(got).detach().double().cpu().reshape(B, -1)
        w = torch.as_tensor(want).detach().double().cpu().reshape(B, -1)
        g, w = g[self.keep], w[self.keep]
        assert torch.isfinite(g).all(), (self.what, name, "unwritten or non-finite rows",
                                         torch.nonzero(~torch.isfinite(g).all(1)).reshape(-1)[:8])
        # each row on the tensor's scale: a row's scalar may itself be a small difference
        err = (g - w).abs().amax(1) / (w.abs().max() + 1e-30)
        e = float(err.max()) if err.numel() else 0.0
        # the first and last row of the ragged last tile, by name in the message
        last0 = (B - 1) // self.R * self.R
        edge = [float(err[i]) for i in (last0, B - 1) if i < err.numel() and bool(self.keep.all())]
        assert e < tol, (self.what, name, "row", int(err.argmax()), e, "last tile", edge)
        self.worst[name] = max(self.worst.get(name, 0.0), e)
        return e

    def whole(self, name, got, want, tol=TOL, scale=None):
        """`scale`: the magnitude of the summed terms when the result is a sum that may cancel
        (a loss over rows, a weight gradient); by default the result's own maximum."""
        g = torch.as_tensor(got).detach().double().cpu().reshape(-1)
        w = torch.as_tensor(want).detach().double().cpu().reshape(-1)
        assert torch.isfinite(g).all(), (self.what, name, g)
        den = w.abs() if scale is None else torch.as_tensor(scale).double().reshape(-1)
        e = float(((g - w).abs() / (den + 1e-30)).max() if scale is not None else
                  (g - w).abs().max() / (w.abs().max() + 1e-30))
        assert e < tol, (self.what, name, e)
        self.worst[name] = max(self.worst.get(name, 0.0), e)
        return e

    def grads(self, name, got, want, dz, inputs, tol):
        """Weight gradients dW_l = dZ_l^T A_l, db_l = sum_b dZ_l, each element on the scale of
        its terms |dZ_l|^T |A_l| (the sums cancel: measured on an H100, an output bias
        gradient over 33 rows came to 5.6e-5 of its own magnitude)."""
        for l, (dW, db) in enumerate(want):
            z, a = dz[l].abs(), inputs[l].abs()
            sw = (z.T @ a).max()
            self.whole(f"{name}.W{l}", got[2 * l], dW, tol, scale=sw.expand(dW.numel()))
            self.whole(f"{name}.b{l}", got[2 * l + 1], db, tol, scale=z.sum(0).max().expand(db.numel()))


def _relu_flips(hidden_k, hidden_64, acts):
    """Rows where a ReLU / leaky-ReLU unit of the kernel sits on the other side of 0 than
    float64 (the oracle follows the kernel's side)."""
    rows = None
    for h, h64, a in zip(hidden_k, hidden_64, acts):
        if a not in ("relu", "leaky_relu"):
            continue
        f = ((h.cpu() > 0) != (h64 > 0)).any(1)
        rows = f if rows is None else rows | f
    return 0 if rows is None else int(rows.sum())


def _h(ws_net):
    return [x.detach().cpu() for x in ws_net.hidden]


# ------------------------------------------------------------------------------------------
# critic step
# ------------------------------------------------------------------------------------------
CRITIC_VARIANTS = ["sac", "sac_single", "td3", "sac_weighted", "td3_weighted", "value_target",
                   "value_target_weighted"]


def _run_critic(case, variant, cfg, B, g, *, regime=None, knife=None):
    """One critic-step launch against ac_fp64.critic_step.  Returns (Cmp or None, oracle)."""
    regime = regime or {}
    algo = "td3" if variant.startswith("td3") else "sac"
    weighted = variant.endswith("weighted") or "weights" in regime
    vt = variant.startswith("value_target")
    single = variant == "sac_single" or regime.get("single")
    actor, q1, q2, v = case.nets(algo, g, regime.get("loc_bias"), regime.get("sl_bias"),
                                 twin_tie=regime.get("twin_tie", False), value=vt,
                                 sl_weight_scale=regime.get("sl_weight_scale"))
    if single:
        q2 = None
    gamma = regime.get("gamma", 0.9)
    if algo == "sac":
        t = _sac(case, actor, q1, q2, v, gamma=gamma, alpha=regime.get("alpha", 0.2))
    else:
        t = _td3(case, actor, q1, q2, gamma=gamma, noise_variance=regime.get("noise_variance", 0.2),
                 noise_clip=regime.get("noise_clip", 0.5))
    b, batch = _batch(case, B, g, regime.get("nan_row"), regime.get("terminal", "mixed"))
    noise = {"next": torch.randn(B, case.A, generator=g) * regime.get("noise_scale", 1.0)}
    _inject(t, noise)
    w = None
    if weighted:
        w = regime.get("weights", lambda B, g: torch.rand(B, generator=g) * 2)(B, g)
    ws = _nan_ws(t, B)
    fill = t._fill_critic if algo == "sac" else t._fill
    fill, bufs = _extra_fill(fill, B, case.A)
    NO = actor["b"][-1].numel()
    hmax = max(case.hmax(), 0)
    R = _tile_rows(cfg, B, case.S + case.A, hmax, _critic_extra(NO))
    tgt1, tgt2 = t._critic_targets() if algo == "sac" else (t.q1_network_target, t.q2_network_target)
    anet = t.actor_network if algo == "sac" else t.actor_network_target
    ok, err = _launch(lambda: t._critic_step(batch, anet, tgt1, tgt2, fill,
                                             sample_weight=None if w is None else w.cuda()))
    what = (repr(case), variant, _cfg_id(cfg), B, sorted(regime))
    if R is None:
        assert not ok and f"rc={E_SMEM}" in err, (what, "a tile that does not fit must be refused")
        assert torch.isnan(ws["td_target"]).all(), (what, "a refused step must not launch")
        return None, None
    assert ok, (what, err)
    fp32 = {"action": bufs["action"].cpu(), "hidden_q1": _h(ws["q1"])}
    if q2 is not None:
        fp32["hidden_q2"] = _h(ws["q2"])
    ref = X.critic_step(actor, q1, q2, q1, q2, b, algo=algo, gamma=gamma,
                        alpha=float(np.float32(regime.get("alpha", 0.2))), noise_next=noise["next"],
                        noise_variance=regime.get("noise_variance", 0.2),
                        noise_clip=regime.get("noise_clip", 0.5), sample_weight=w,
                        value_target=v, fp32=fp32)
    nan_row = regime.get("nan_row")
    c = Cmp(B, R, what, skip_rows=nan_row)
    fwd = case.chain()
    c.rows("td_target", ws["td_target"], ref["td_target"], fwd)
    c.rows("q1_value", ws["q1_value"], ref["q1_value"], fwd)
    c.rows("input", ws["q1"].input, ref["input"])
    if not vt:
        c.rows("next_action", bufs["action"], ref["next_action"], fwd)
        if algo == "sac":
            c.rows("log_prob", ws["log_prob"], ref["log_prob"], fwd)
    if w is not None:
        c.rows("td_error", ws["td_error"], ref["td_error"], fwd)
    ks = ["q1"] + ([] if q2 is None else ["q2"])
    if q2 is not None:
        c.rows("q2_value", ws["q2_value"], ref["q2_value"], fwd)
    for k in ks:
        for l, (h, h64) in enumerate(zip(ws[k].hidden, ref["hidden_" + k])):
            c.rows(f"hidden_{k}{l}", h, h64, _tol(max([case.S + case.A] + case.sizes)))
        for l, (dz, dz64) in enumerate(zip(ws[k].dz, ref["dz_" + k])):
            c.rows(f"dz_{k}{l}", dz, dz64, fwd)
    if nan_row is not None:
        assert torch.isnan(ws["td_error"][nan_row]).all(), (what, "NaN reward -> NaN TD error")
        assert torch.isnan(ws["critic_loss"][:len(ks)]).all(), (what, "NaN reward -> NaN loss")
    else:
        c.whole("loss", ws["critic_loss"][:len(ks)], ref["loss"], max(fwd, _tol(B)),
                scale=ref["loss_scale"])
        for k in ks:
            net = t.q1_network if k == "q1" else t.q2_network
            c.grads("grad_" + k, t.net_grads(net), ref["grad_" + k], ref["dz_" + k],
                    [ref["input"]] + ref["hidden_" + k], max(fwd, _tol(B)))
    if knife is not None:
        flips = sum(_relu_flips(_h(ws[k]), ref["hidden_" + k], case.acts) for k in ks)
        if not vt and algo == "sac":
            a64 = ref["next_action"]
            flips += int(((a64.abs() < X.ACT_HI) != (bufs["action"].cpu().double().abs() < X.ACT_HI))
                         .any(1).sum())
        knife.append(flips)
    return c, ref


@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
@pytest.mark.parametrize("variant", CRITIC_VARIANTS)
def test_critic_step_matches_fp64(monkeypatch, cfg, variant):
    _set_cfg(monkeypatch, cfg)
    worst, knife, launched = {}, [], 0
    for ci, case in enumerate(CASES):
        g = torch.Generator().manual_seed(1000 * ci + CRITIC_VARIANTS.index(variant))
        for B in case.batches:
            c, _ = _run_critic(case, variant, cfg, B, g, knife=knife)
            if c is None:
                continue
            launched += 1
            for k, e in c.worst.items():
                worst[k] = max(worst.get(k, 0.0), e)
    assert launched > 0, "no shape fits this tile"
    assert max(knife) <= MAX_KNIFE_EDGE_ROWS, knife
    _record("ac_critic_step", variant=variant, cfg=_cfg_id(cfg), launched=launched,
            knife_edge_rows=sum(knife), worst=worst)


# ------------------------------------------------------------------------------------------
# actor step
# ------------------------------------------------------------------------------------------
ACTOR_VARIANTS = ["sac", "sac_single", "sac_no_logprob_grad", "td3", "crr_indicator",
                  "crr_exponent"]


def _run_actor(case, variant, cfg, B, g, *, regime=None, knife=None):
    regime = regime or {}
    algo = "td3" if variant == "td3" else "sac"
    crr = None
    if variant == "crr_indicator":
        crr = {"indicator_fn_threshold": regime.get("threshold", 0.1)}
    elif variant == "crr_exponent":
        crr = {"exponent_beta": regime.get("beta", 0.5), "exponent_clamp": regime.get("clamp", 2.0)}
    nets = regime.get("nets")
    if nets is None:
        actor, q1, q2, v = case.nets(algo, g, regime.get("loc_bias"), regime.get("sl_bias"),
                                     twin_tie=regime.get("twin_tie", False), value=crr is not None,
                                     sl_weight_scale=regime.get("sl_weight_scale"))
    else:
        actor, q1, q2, v = nets(case, g)
    if variant == "sac_single":
        q2 = None
    if "q_shift" in regime:
        for n in (q1, q2):
            n["b"][-1] += regime["q_shift"]
    alpha, te = regime.get("alpha", 0.2), -float(case.A)
    if algo == "sac":
        t = _sac(case, actor, q1, q2, v, alpha=alpha, target_entropy=te,
                 backprop=variant != "sac_no_logprob_grad", crr=crr)
    else:
        t = _td3(case, actor, q1, q2)
    b, batch = _batch(case, B, g)
    if "state" in regime:
        b["state"] = regime["state"](b["state"], g)
        batch = _pbatch({k: v_.cuda() for k, v_ in b.items()})
    noise = {"cur": torch.randn(B, case.A, generator=g) * regime.get("noise_scale", 1.0)}
    _inject(t, noise)
    ws = _nan_ws(t, B)
    fill = t._fill_actor if algo == "sac" else t._fill
    fill, bufs = _extra_fill(fill, B, case.A, want_min_q=v is None)
    NO = actor["b"][-1].numel()
    hmax = max(case.hmax(), 0)
    R = _tile_rows(cfg, B, case.S + case.A, hmax, _actor_extra(NO))
    ok, err = _launch(lambda: t._actor_step(batch, fill))
    what = (repr(case), variant, _cfg_id(cfg), B, sorted(k for k in regime if k != "nets"))
    if R is None:
        assert not ok and f"rc={E_SMEM}" in err, (what, "a tile that does not fit must be refused")
        assert torch.isnan(ws["actor"].dz[0]).all(), (what, "a refused step must not launch")
        return None, None
    assert ok, (what, err)
    min_q = bufs["min_q"] if v is None else ws["min_q"]
    fp32 = {"action": bufs["action"].cpu(), "hidden_actor": _h(ws["actor"]),
            "hidden_q1": _h(ws["q1"])}
    use_q2 = algo == "sac" and q2 is not None
    if use_q2:
        fp32["hidden_q2"] = _h(ws["q2"])
    if algo == "sac":
        fp32["log_prob"] = ws["log_prob"].cpu()
    la = float(t.log_alpha.detach()) if algo == "sac" else None
    ref = X.actor_step(actor, q1, q2, b, algo=algo, alpha=float(np.float32(alpha)), log_alpha=la,
                       target_entropy=te, noise_cur=noise["cur"],
                       backprop_through_log_prob=variant != "sac_no_logprob_grad", value_net=v,
                       crr=crr, fp32=fp32)
    c = Cmp(B, R, what)
    fwd = case.chain()
    c.rows("action", bufs["action"], ref["action"], fwd)
    c.rows("min_q", min_q, ref["min_q"], fwd)
    if algo == "sac":
        c.rows("log_prob", ws["log_prob"], ref["log_prob"], fwd)
    for l, (h, h64) in enumerate(zip(ws["actor"].hidden, ref["hidden_actor"])):
        c.rows(f"hidden_actor{l}", h, h64, _tol(max([case.S] + case.sizes)))
    for k in ["q1"] + (["q2"] if use_q2 else []):
        for l, (h, h64) in enumerate(zip(ws[k].hidden, ref["hidden_" + k])):
            c.rows(f"hidden_{k}{l}", h, h64, _tol(max([case.S + case.A] + case.sizes)))
    for l, (dz, dz64) in enumerate(zip(ws["actor"].dz, ref["dz_actor"])):
        c.rows(f"dz_actor{l}", dz, dz64, fwd)
    c.whole("loss", ws["actor_loss"][0], ref["loss"], max(fwd, _tol(B)), scale=ref["loss_scale"])
    if algo == "sac":
        c.whole("alpha_grad", ws["alpha_grad"], ref["alpha_grad"], _tol(B))
        c.whole("alpha_loss", ws["actor_loss"][1], ref["alpha_loss"], _tol(B))
    c.grads("grad_actor", t.net_grads(t.actor_network), ref["grad_actor"], ref["dz_actor"],
            [X._d(b["state"])] + ref["hidden_actor"], max(fwd, _tol(B)))
    if knife is not None:
        ks = ["actor", "q1"] + (["q2"] if use_q2 else [])
        flips = sum(_relu_flips(_h(ws[k]), ref["hidden_" + k], case.acts) for k in ks)
        if algo == "sac":
            a64 = ref["action"]
            flips += int(((a64.abs() < X.ACT_HI) != (bufs["action"].cpu().double().abs() < X.ACT_HI))
                         .any(1).sum())
            lp64, lpk = ref["log_prob"], ws["log_prob"].cpu().double()
            flips += int((((lp64 >= -2) & (lp64 <= 2)) != ((lpk >= -2) & (lpk <= 2))).sum())
        knife.append(flips)
    return c, ref


@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
@pytest.mark.parametrize("variant", ACTOR_VARIANTS)
def test_actor_step_matches_fp64(monkeypatch, cfg, variant):
    _set_cfg(monkeypatch, cfg)
    worst, knife, launched = {}, [], 0
    for ci, case in enumerate(CASES):
        g = torch.Generator().manual_seed(2000 * ci + ACTOR_VARIANTS.index(variant))
        for B in case.batches:
            c, _ = _run_actor(case, variant, cfg, B, g, knife=knife)
            if c is None:
                continue
            launched += 1
            for k, e in c.worst.items():
                worst[k] = max(worst.get(k, 0.0), e)
    assert launched > 0, "no shape fits this tile"
    assert max(knife) <= MAX_KNIFE_EDGE_ROWS, knife
    _record("ac_actor_step", variant=variant, cfg=_cfg_id(cfg), launched=launched,
            knife_edge_rows=sum(knife), worst=worst)


# ------------------------------------------------------------------------------------------
# value step
# ------------------------------------------------------------------------------------------
def _run_value(case, cfg, B, g, uniform_prior):
    actor, q1, q2, v = case.nets("sac", g, value=True)
    t = _sac(case, actor, q1, q2, v, alpha=0.3, uniform_prior=uniform_prior)
    b, batch = _batch(case, B, g)
    ws = _nan_ws(t, B)
    # the actor step's outputs the value step reads; log-probs beyond both clamp ends
    min_q = torch.randn(B, generator=g)
    lp = torch.randn(B, generator=g) * 4
    ws["min_q"].copy_(min_q)
    ws["log_prob"].copy_(lp)
    R = _tile_rows(cfg, B, case.S, case.hmax(), 9)
    ok, err = _launch(lambda: t._value_step(batch))
    what = (repr(case), "value", _cfg_id(cfg), B, uniform_prior)
    if R is None:
        assert not ok and f"rc={E_SMEM}" in err, (what, "a tile that does not fit must be refused")
        assert torch.isnan(ws["value"].dz[0]).all(), (what, "a refused step must not launch")
        return None
    assert ok, (what, err)
    ref = X.value_step(v, b["state"], min_q, log_prob=lp, alpha=float(np.float32(0.3)),
                       logged_action_uniform_prior=uniform_prior,
                       fp32={"hidden_value": _h(ws["value"])})
    c = Cmp(B, R, what)
    for l, (h, h64) in enumerate(zip(ws["value"].hidden, ref["hidden"])):
        c.rows(f"hidden{l}", h, h64, _tol(max([case.S] + case.sizes)))
    for l, (dz, dz64) in enumerate(zip(ws["value"].dz, ref["dz"])):
        c.rows(f"dz{l}", dz, dz64, case.chain())
    c.whole("loss", ws["value_loss"], ref["loss"], max(case.chain(), _tol(B)))
    c.grads("grad", t.net_grads(t.value_network), ref["grad"], ref["dz"],
            [X._d(b["state"])] + ref["hidden"], max(case.chain(), _tol(B)))
    return c


@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
@pytest.mark.parametrize("uniform_prior", [True, False])
def test_value_step_matches_fp64(monkeypatch, cfg, uniform_prior):
    _set_cfg(monkeypatch, cfg)
    worst, launched = {}, 0
    for ci, case in enumerate(CASES):
        g = torch.Generator().manual_seed(3000 * ci + uniform_prior)
        for B in case.batches:
            c = _run_value(case, cfg, B, g, uniform_prior)
            if c is None:
                continue
            launched += 1
            for k, e in c.worst.items():
                worst[k] = max(worst.get(k, 0.0), e)
    assert launched > 0
    _record("ac_value_step", cfg=_cfg_id(cfg), uniform_prior=uniform_prior, launched=launched,
            worst=worst)


# ------------------------------------------------------------------------------------------
# forced regimes
# ------------------------------------------------------------------------------------------
REGIME_CASE = Case(8, 3, [64, 32], ["relu", "tanh"])
REGIME_BATCHES = (17, 33)


def _weights_with_extremes(B, g):
    w = torch.rand(B, generator=g) * 2
    w[::5] = 0.0
    w[1::7] = 1e4
    return w


CRITIC_REGIMES = {
    # scale_log beyond each end of [-2, 2], actions deep in tanh saturation
    "sl_high_saturated": ("sac", {"loc_bias": [15.0, -15.0, 15.0], "sl_bias": 8.0,
                                  "noise_scale": 0.1}),
    "sl_low_saturated": ("sac", {"loc_bias": [-15.0, 15.0, 12.0], "sl_bias": -8.0}),
    # every target row a twin tie
    "twin_tie": ("sac", {"twin_tie": True}),
    # draws far beyond the clip and target actions beyond +-1
    "td3_noise_clip": ("td3", {"noise_scale": 10.0, "noise_variance": 0.2, "noise_clip": 0.3}),
    "gamma_zero": ("sac", {"gamma": 0.0}),
    "gamma_negative": ("sac", {"gamma": -0.5}),
    "all_terminal": ("sac", {"terminal": "all"}),
    "td3_all_terminal": ("td3", {"terminal": "all", "gamma": 0.0}),
    "value_target_gamma_negative": ("value_target", {"gamma": -0.5}),
    "weights_and_nan_reward": ("sac", {"weights": _weights_with_extremes, "nan_row": 3}),
    "td3_weights_and_nan_reward": ("td3", {"weights": _weights_with_extremes, "nan_row": 0}),
}


@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
@pytest.mark.parametrize("regime", sorted(CRITIC_REGIMES))
def test_critic_step_regimes(monkeypatch, cfg, regime):
    _set_cfg(monkeypatch, cfg)
    variant, reg = CRITIC_REGIMES[regime]
    worst = {}
    for B in REGIME_BATCHES:
        g = torch.Generator().manual_seed(B)
        knife = []
        c, ref = _run_critic(REGIME_CASE, variant, cfg, B, g, regime=reg, knife=knife)
        if c is None:
            continue
        assert knife == [0], (regime, knife)
        # the regime is reached
        if "sl_bias" in reg:
            assert (ref["next_action"].abs() == X.ACT_HI).all()
            lp = ref["log_prob"]
            assert ((lp > 2) | (lp < -2)).all(), lp
        if regime == "td3_noise_clip":
            assert (ref["next_action"].abs() == 1.0).any() and (ref["next_action"].abs() < 1).any()
        for k, e in c.worst.items():
            worst[k] = max(worst.get(k, 0.0), e)
    _record("ac_critic_regime", regime=regime, cfg=_cfg_id(cfg), worst=worst)


def _crr_tie_nets(case, g):
    """Single-hidden-layer ReLU nets whose hidden layer is all zero on rows with state 0 (the
    first-layer biases are below -sum|W| over the action columns): there q1 = 0.75, q2 = 1.75
    and V = 0.25 exactly, so adv = min_q - V = 0.5, the indicator's threshold, to the bit."""
    S, A, H = case.S, case.A, case.sizes[0]
    actor = _net([S, H, 2 * A], ["relu", "linear"], g)
    q1 = _net([S + A, H, 1], ["relu", "linear"], g)
    q2 = _net([S + A, H, 1], ["relu", "linear"], g)
    v = _net([S, H, 1], ["relu", "linear"], g)
    for n, b in ((q1, 0.75), (q2, 1.75), (v, 0.25)):
        n["b"][0] = -2.0 - n["W"][0][:, S:].abs().sum(1) - torch.rand(H, generator=g)
        n["b"][1] = torch.tensor([b])
    return actor, q1, q2, v


def _zero_some_states(s, g):
    s = s * 3.0
    s[::3] = 0.0
    return s


CRR_TIE_CASE = Case(8, 3, [32], ["relu"])
BAND_CASE = Case(8, 4, [64, 32], ["relu", "tanh"])


def _tie_distinct_grads_nets(case, g):
    """pi(s) = 0 exactly (loc weights and bias 0, zero noise), and q2 is q1 with other weights
    on the action columns: q1(s, 0) == q2(s, 0) to the bit on every row, while their action
    gradients differ, so the 0.5 / 0.5 split of the tie shows in the actor's dZ."""
    actor, q1, _, _ = case.nets("sac", g)
    actor["W"][-1][:case.A] = 0.0
    actor["b"][-1][:case.A] = 0.0
    q2 = {"W": [w.clone() for w in q1["W"]], "b": [b.clone() for b in q1["b"]], "act": q1["act"]}
    q2["W"][0][:, case.S:] = torch.randn(q2["W"][0][:, case.S:].shape, generator=g)
    return actor, q1, q2, None


def _clamp_band_nets(case, g):
    """Action 0 clamped with tanh(raw) still below 1 in fp32 (raw ~ 8: the band between the
    bound 1 - 1.013e-6 and fp32's 1.0, where only the clamp mask zeroes its gradient), and
    the summed log-prob inside [-2, 2] so that gradient is not zero anyway."""
    actor, q1, q2, _ = case.nets("sac", g)
    actor["W"][-1].zero_()
    actor["b"][-1] = torch.tensor([8.0] + [0.0] * (case.A - 1) + [1.9] * case.A)
    return actor, q1, q2, None

ACTOR_REGIMES = {
    "sl_high_saturated": ("sac", REGIME_CASE, {"loc_bias": [15.0, -15.0, 15.0], "sl_bias": 8.0,
                                               "noise_scale": 0.1}),
    "sl_low_saturated": ("sac", REGIME_CASE, {"loc_bias": [-15.0, 15.0, 12.0], "sl_bias": -8.0}),
    "sl_low_unsaturated": ("sac", REGIME_CASE, {"loc_bias": 0.0, "sl_bias": -8.0}),
    "twin_tie": ("sac", REGIME_CASE, {"twin_tie": True}),
    "twin_tie_saturated": ("sac", REGIME_CASE, {"twin_tie": True, "loc_bias": 15.0,
                                                "sl_bias": -8.0}),
    "twin_tie_distinct_grads": ("sac", REGIME_CASE, {"nets": _tie_distinct_grads_nets,
                                                     "noise_scale": 0.0}),
    "clamp_band": ("sac", BAND_CASE, {"nets": _clamp_band_nets, "noise_scale": 0.01}),
    "crr_indicator_at_threshold": ("crr_indicator", CRR_TIE_CASE,
                                   {"nets": _crr_tie_nets, "state": _zero_some_states,
                                    "threshold": 0.5}),
    # adv ~ 10, adv / beta ~ 200: exp overflows fp32 on every row and the clamp caps it
    "crr_exponent_overflow_clamped": ("crr_exponent", REGIME_CASE,
                                      {"beta": 0.05, "clamp": 3.0, "q_shift": 10.0}),
    "crr_exponent_unclamped": ("crr_exponent", REGIME_CASE, {"beta": 4.0, "clamp": None}),
}


@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
@pytest.mark.parametrize("regime", sorted(ACTOR_REGIMES))
def test_actor_step_regimes(monkeypatch, cfg, regime):
    _set_cfg(monkeypatch, cfg)
    variant, case, reg = ACTOR_REGIMES[regime]
    worst = {}
    for B in REGIME_BATCHES:
        g = torch.Generator().manual_seed(B)
        knife = []
        c, ref = _run_actor(case, variant, cfg, B, g, regime=reg, knife=knife)
        if c is None:
            continue
        assert knife == [0], (regime, knife)
        lp = ref.get("log_prob")
        if "saturated" in regime and "unsaturated" not in regime:
            assert (ref["action"].abs() == X.ACT_HI).all()
        if "saturated" in regime and "unsaturated" not in regime:
            assert ((lp > 2) | (lp < -2)).all(), lp
        if regime == "twin_tie_distinct_grads":
            assert (ref["action"] == 0).all()
        if regime == "clamp_band":
            a0 = ref["action"][:, 0]
            assert (a0 == X.ACT_HI).all() and ((lp >= -2) & (lp <= 2)).all(), lp
        if regime == "crr_exponent_overflow_clamped":
            assert (ref["min_q"] > 0.05 * 89).all()      # exp(adv / beta) > FLT_MAX
        if regime == "crr_indicator_at_threshold":
            ties = (ref["min_q"] - 0.25) == 0.5
            assert ties.sum() >= B // 3, int(ties.sum())
        for k, e in c.worst.items():
            worst[k] = max(worst.get(k, 0.0), e)
    _record("ac_actor_regime", regime=regime, cfg=_cfg_id(cfg), worst=worst)


# ------------------------------------------------------------------------------------------
# the benchmark's shapes, on the tile the library picks for them
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("config", [4, 5])
def test_bench_shape_matches_fp64(monkeypatch, config):
    """bench.py --gpus 1: config 4 (SAC, S 256, A 32, [256, 256], B 8192) and config 5 (TD3,
    S 512, A 64, B 16384), both above 2112 rows, so the 32-row tiles run."""
    _set_cfg(monkeypatch, None)
    S, A, B, algo = (256, 32, 8192, "sac") if config == 4 else (512, 64, 16384, "td3")
    case = Case(S, A, [256, 256], ["relu", "relu"])
    NO = 2 * A if algo == "sac" else A
    assert _pick(None, B, S + A, 256, 1, 3, _critic_extra(NO))[0] == 512
    g = torch.Generator().manual_seed(config)
    knife = []
    # 262144 scale_log values would put some within fp32 noise of the clamp at +-2, where the
    # mask (not observable in the workspace) decides a whole dZ element: keep them O(0.2)
    reg = {"sl_weight_scale": 0.2}
    c, _ = _run_critic(case, algo, None, B, g, regime=reg, knife=knife)
    worst = dict(c.worst)
    ca, _ = _run_actor(case, algo, None, B, g, regime=reg, knife=knife)
    worst.update({"actor." + k: e for k, e in ca.worst.items()})
    # 256-wide ReLU layers at 8192 rows: measured 18 rows with a unit within fp32 noise of 0
    assert max(knife) <= MAX_KNIFE_EDGE_ROWS + B // 200, knife
    _record("ac_bench_shape", config=config, B=B, knife_edge_rows=knife, worst=worst)
