"""TEST INFRASTRUCTURE ONLY -- float64 restatements of the three fused actor-critic launches
(rb200_ac_critic_step, rb200_ac_actor_step, rb200_ac_value_step) for one batch, on float64
copies of the exact fp32 weights, inputs and injected noise.

Each function restates the reference lines it cites and returns what its launch writes: the
per-row outputs, the losses, the dZ of every layer (d loss / d pre-activation, from
torch.autograd in float64), the saved hidden activations and the parameter gradients.
tests/test_ac_fp64_cpu.py pins them against oracle/td_oracle.py, oracle/per_ac_oracle.py and
oracle/sac_value_oracle.py (themselves pinned to the unmodified reference);
tests/test_ac_kernels_gpu.py compares the CUDA kernels with them in every row-tile
configuration.

Networks are td_oracle's {"W": [...], "b": [...], "act": [...]} dicts.  Three fp32 facts of
the reference are mirrored, so that what remains is the kernel's own error:

* The clamp bounds are fp32 numbers: the reference clamps fp32 tensors, so the action bound is
  float32(1 - 1e-6) = 1 - 1.013e-6, not 1 - 1e-6.  Every bound is taken as its fp32 value.
* The squash correction log(1 - a**2 + 1e-6) squares the fp32 action in fp32.  At a saturated
  action 1 - a**2 is ~2e-6, so that rounding moves the log-prob by up to ~1e-4; the value
  mirrors it (the derivative is the exact one).
* get_log_prob recomputes the log-prob from the fp32 squashed action, where atanh is
  ill-conditioned.  The caller may pass the kernel's fp32 actions (`fp32["action"]`); the
  log-prob, the critics downstream and the tanh / clamp backward are then evaluated in float64
  from exactly those actions, while `action` in the result stays the float64 tanh to check
  them against.

Optional `fp32` entries feed the kernel's fp32 decisions back in the same way: "hidden_*"
(saved activations: the activation derivatives are taken from them, as the kernels take them,
so a unit within fp32 noise of a ReLU kink cannot flip), "log_prob" (the log-prob clamp mask).
Each of these must itself be checked against the float64 value the function returns."""
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

f64 = torch.float64


def f32(x: float) -> float:
    """x rounded to the nearest fp32 number (the value a bound takes on an fp32 tensor)."""
    return float(np.float32(x))


LOG_PROB_MIN, LOG_PROB_MAX = -2.0, 2.0          # reagent/models/actor.py:18-19 (exact in fp32)
ACT_EPS = f32(1e-6)                             # actor.py:165
ACT_HI = f32(1.0 - 1e-6)                        # clamp(tanh(raw), -1 + eps, 1 - eps)
ACT_LO = f32(-1.0 + 1e-6)
LOG_SQRT_2PI = float(np.log(np.sqrt(2 * np.pi)))


def _d(x):
    return None if x is None else torch.as_tensor(x).detach().to("cpu", f64)


def _act(z, act):
    if act == "relu":
        return torch.relu(z)
    if act == "tanh":
        return torch.tanh(z)
    if act == "leaky_relu":
        return F.leaky_relu(z, 0.01)
    if act == "sigmoid":
        return torch.sigmoid(z)
    if act == "softplus":
        return F.softplus(z)
    assert act == "linear", act
    return z


def dact_from_out(h, act):
    """act'(z) through the activation's output h, as the kernels (and torch's relu / tanh /
    sigmoid backward) evaluate it."""
    if act == "relu":
        return (h > 0).to(f64)
    if act == "leaky_relu":
        return torch.where(h > 0, 1.0, 0.01).to(f64)
    if act == "tanh":
        return 1.0 - h * h
    if act == "sigmoid":
        return h * (1.0 - h)
    if act == "softplus":
        return 1.0 - torch.exp(-h)
    return torch.ones_like(h)


class _ActOut(torch.autograd.Function):
    """act(z) in float64 whose backward takes act' from `h_ext` (fp32 activations the kernel
    saved) instead of from its own output."""

    @staticmethod
    def forward(ctx, z, h_ext, act):
        ctx.act = act
        ctx.save_for_backward(h_ext)
        return _act(z, act)

    @staticmethod
    def backward(ctx, g):
        (h,) = ctx.saved_tensors
        return g * dact_from_out(h, ctx.act), None, None


def _act_ext(z, act, h_ext):
    if h_ext is None or act == "linear":
        return _act(z, act)
    return _ActOut.apply(z, _d(h_ext).reshape(z.shape), act)


class Net64:
    """A float64, gradient-tracking copy of one network."""

    def __init__(self, net):
        self.W = [_d(w).clone().requires_grad_(True) for w in net["W"]]
        self.b = [_d(b).clone().requires_grad_(True) for b in net["b"]]
        self.act = list(net["act"])

    def params(self):
        out = []
        for w, b in zip(self.W, self.b):
            out += [w, b]
        return out

    def forward(self, x, hidden_ext=None, last_ext=None):
        """(output, [pre-activations], [hidden activations]) of FullyConnectedNetwork.forward
        (reagent/models/fully_connected_network.py:157-163)."""
        zs, hs, h = [], [], x
        L = len(self.act)
        for l in range(L):
            z = h @ self.W[l].T + self.b[l]
            ext = last_ext if l == L - 1 else (None if hidden_ext is None else hidden_ext[l])
            h = _act_ext(z, self.act[l], ext)
            zs.append(z)
            if l < L - 1:
                hs.append(h)
        return h, zs, hs


def _grads(loss, nets_zs):
    """autograd of `loss` w.r.t. each (Net64, zs): {"dz": [...], "grad": [(dW, db)...]}."""
    flat = []
    for net, zs in nets_zs:
        flat += list(zs) + net.params()
    g = torch.autograd.grad(loss, flat, allow_unused=True, retain_graph=True)
    out, k = [], 0
    for net, zs in nets_zs:
        dz = [torch.zeros_like(z) if t is None else t.detach() for z, t in zip(zs, g[k:k + len(zs)])]
        k += len(zs)
        ps = g[k:k + 2 * len(net.W)]
        k += 2 * len(net.W)
        out.append({"dz": dz, "grad": [(ps[2 * i].detach(), ps[2 * i + 1].detach())
                                       for i in range(len(net.W))]})
    return out


def _round32(x):
    return x.detach().to(torch.float32).to(f64)


def _straight(value, x):
    """`value` forward, d/dx backward (value fixed, gradient through x's graph)."""
    return x + (value - x).detach()


def gaussian_head(out, noise, fp32_action=None, fp32_log_prob=None):
    """GaussianFullyConnectedActor.forward + get_log_prob (reagent/models/actor.py:202-261) on
    the actor output `out` [B, 2A]: returns (squashed action (float64 tanh, clamped),
    action the rest uses (= fp32_action in value when given), log_prob [B] unclamped,
    log-prob clamp mask [B])."""
    A = out.shape[1] // 2
    loc, slr = out[:, :A], out[:, A:]
    sl = slr.clamp(LOG_PROB_MIN, LOG_PROB_MAX)
    sigma = sl.exp()
    raw = loc + _d(noise) * sigma
    if fp32_action is None:
        t = torch.tanh(raw)
        in_range = (t >= ACT_LO) & (t <= ACT_HI)
        a_own = t.clamp(ACT_LO, ACT_HI)
        a = a_own
    else:
        ak = _d(fp32_action)
        # tanh backward through the fp32 output, as torch's tanh_backward takes it
        t = _ActOut.apply(raw, ak, "tanh")
        # clamp backward where the fp32 action is strictly inside the bounds
        in_range = (ak > ACT_LO) & (ak < ACT_HI)
        a_own = torch.tanh(raw.detach()).clamp(ACT_LO, ACT_HI)
        a = _straight(ak, torch.where(in_range, t, t.detach()))
    r = (torch.atanh(a) - loc) / sigma
    a2 = a * a
    corr_exact = torch.log(1.0 - a2 + ACT_EPS)
    corr = _straight(torch.log(1.0 - _round32(a2) + ACT_EPS), corr_exact)
    lp = (-(r * r) / 2 - sl - LOG_SQRT_2PI - corr).sum(1)
    lpm = lp.detach() if fp32_log_prob is None else _d(fp32_log_prob).reshape(-1)
    lp_in = (lpm >= LOG_PROB_MIN) & (lpm <= LOG_PROB_MAX)
    return a_own.detach(), a, lp, lp_in


def _clamp_lp(lp, lp_in):
    """clamp(log_prob, -2, 2) whose backward mask is `lp_in`."""
    c = lp.clamp(LOG_PROB_MIN, LOG_PROB_MAX)
    return torch.where(lp_in, lp, c.detach())


def _get(fp32, key):
    return None if fp32 is None else fp32.get(key)


def critic_step(actor, q1, q2, q1t, q2t, batch, *, algo, gamma, alpha=None, noise_next=None,
                noise_variance=None, noise_clip=None, sample_weight=None, value_target=None,
                fp32=None):
    """rb200_ac_critic_step: SAC sac_trainer.py:214-248, TD3 td3_trainer.py:138-178 (with
    `value_target`: sac_trainer.py:214-217, V'(s') replaces the actor and the q targets).
    `batch`: state, action, next_state, reward, not_terminal.  `fp32`: "action" (the kernel's
    next_action_out), "hidden_q1" / "hidden_q2".  Returns next_action, log_prob, td_target,
    q1_value, q2_value, loss [2], td_error (weighted), and per critic k in (q1, q2):
    dz_k, hidden_k, grad_k; input (the critics' cat(state, action))."""
    s, act = _d(batch["state"]), _d(batch["action"])
    ns = _d(batch["next_state"])
    B = s.shape[0]
    reward, nt = _d(batch["reward"]).reshape(B), _d(batch["not_terminal"]).reshape(B)
    out = {}
    with torch.no_grad():
        if value_target is not None:
            nsv = Net64(value_target).forward(ns)[0].reshape(B)
            tgt = reward + gamma * nsv * nt if gamma > 0.0 else reward       # :233-239
        else:
            aout = Net64(actor).forward(ns)[0]
            if algo == "sac":
                a_own, a_next, lp, _ = gaussian_head(aout, noise_next, _get(fp32, "action"))
                out["log_prob"] = lp
            else:                                                           # td3_trainer.py:139-144
                n = (_d(noise_next) * f32(noise_variance)).clamp(-f32(noise_clip), f32(noise_clip))
                a_own = (aout + n).clamp(-1.0, 1.0)
                a_next = a_own if _get(fp32, "action") is None else _d(fp32["action"])
            out["next_action"] = a_own
            cin = torch.cat([ns, a_next], 1)
            nsv = Net64(q1t).forward(cin)[0].reshape(B)
            if q2 is not None:
                nsv = torch.minimum(nsv, Net64(q2t).forward(cin)[0].reshape(B))
            if algo == "sac":
                nsv = nsv - float(alpha) * lp.clamp(LOG_PROB_MIN, LOG_PROB_MAX)  # :228-231
                tgt = reward + gamma * nsv * nt if gamma > 0.0 else reward       # :233-239
            else:
                tgt = reward + gamma * nsv * nt
    out["td_target"] = tgt
    x = torch.cat([s, act], 1)
    out["input"] = x
    w = None if sample_weight is None else _d(sample_weight).reshape(B)
    losses, scales, td_err = [], [], None
    for k, q in (("q1", q1), ("q2", q2)):
        if q is None:
            continue
        net = Net64(q)
        qv, zs, hs = net.forward(x, _get(fp32, "hidden_" + k))
        qv = qv.reshape(B)
        d = qv - tgt
        le = d * d if w is None else w * (d * d)
        loss = le.mean()                                  # F.mse_loss / mean(w * (q - y)^2)
        g = _grads(loss, [(net, zs)])[0]
        e = d.detach().abs()
        td_err = e if td_err is None else torch.maximum(td_err, e)
        out[k + "_value"] = qv.detach()
        out["dz_" + k], out["grad_" + k] = g["dz"], g["grad"]
        out["hidden_" + k] = [h.detach() for h in hs]
        losses.append(loss.detach())
        scales.append(le.detach().abs().mean())
    out["loss"] = torch.stack(losses)
    out["loss_scale"] = torch.stack(scales)     # mean |per-row term|: the loss's own scale
    if w is not None:
        out["td_error"] = td_err
    return out


def actor_step(actor, q1, q2, batch, *, algo, alpha=None, log_alpha=None, target_entropy=None,
               noise_cur=None, backprop_through_log_prob=True, value_net=None, crr=None,
               fp32=None):
    """rb200_ac_actor_step: SAC sac_trainer.py:254-322 (alpha loss included; CRR weighting
    :265-276 when `crr` = dict(indicator_fn_threshold= | exponent_beta=, exponent_clamp=) with
    `value_net`), TD3 td3_trainer.py:181-187 (q1 only).  `fp32`: "action" (the kernel's
    pi(s)), "log_prob", "hidden_actor", "hidden_q1", "hidden_q2".  Returns action, log_prob,
    min_q, loss, alpha_grad, alpha_loss, dz_actor, hidden_actor, grad_actor, hidden_q1,
    hidden_q2."""
    s = _d(batch["state"])
    B = s.shape[0]
    anet = Net64(actor)
    sac = algo == "sac"
    if sac:
        aout, zs, hs = anet.forward(s, _get(fp32, "hidden_actor"))
        a_own, a, lp, lp_in = gaussian_head(aout, noise_cur, _get(fp32, "action"),
                                            _get(fp32, "log_prob"))
    else:
        a, zs, hs = anet.forward(s, _get(fp32, "hidden_actor"), last_ext=_get(fp32, "action"))
        a_own = a.detach()
    out = {"action": a_own, "hidden_actor": [h.detach() for h in hs]}
    x = torch.cat([s, a], 1)
    use_q2 = sac and q2 is not None
    qs = []
    for k, q in (("q1", q1), ("q2", q2 if use_q2 else None)):
        if q is None:
            continue
        qv, _, qh = Net64(q).forward(x, _get(fp32, "hidden_" + k))
        qs.append(qv.reshape(B))
        out["hidden_" + k] = [h.detach() for h in qh]
    if use_q2:
        # torch.min(a, b) backward: ties split the gradient evenly
        w1 = (qs[0] < qs[1]).to(f64) + 0.5 * (qs[0] == qs[1]).to(f64)
        minq = w1.detach() * qs[0] + (1.0 - w1.detach()) * qs[1]
    else:
        minq = qs[0]
    out["min_q"] = minq.detach()
    if sac:
        lpc = _clamp_lp(lp, lp_in)
        out["log_prob"] = lp.detach()
        if crr is not None:
            adv = (minq - Net64(value_net).forward(s)[0].reshape(B)).detach()
            if crr.get("indicator_fn_threshold"):
                wt = (adv >= crr["indicator_fn_threshold"]).to(f64)
            else:
                wt = torch.exp(adv / crr["exponent_beta"])
                # fp32 exp overflows to inf beyond log(FLT_MAX); the clamp then caps it
                wt = torch.where(wt > float(np.finfo(np.float32).max), float("inf"), wt)
                if crr.get("exponent_clamp"):
                    wt = wt.clamp(0.0, crr["exponent_clamp"])
            rows = -(lpc * wt)
            loss = rows.mean()                                               # :265-276
            mag = lp.detach().abs() * wt
        else:
            lpt = lpc if backprop_through_log_prob else lpc.detach()
            rows = float(alpha) * lpt - minq
            loss = rows.mean()                                               # :278
            mag = float(alpha) * lp.detach().abs() + minq.detach().abs()
        m = (lp.detach().clamp(LOG_PROB_MIN, LOG_PROB_MAX) + target_entropy).mean()
        out["alpha_grad"] = -m                                               # :311-322
        out["alpha_loss"] = None if log_alpha is None else -(float(log_alpha) * m)
    else:
        rows = -minq
        loss = rows.mean()                                                   # td3_trainer.py:184
        mag = minq.detach().abs()
    g = _grads(loss, [(anet, zs)])[0]
    out["loss"] = loss.detach()
    # the largest per-row magnitude behind the loss (rows are exact to their tensor's scale)
    out["loss_scale"] = mag.max()
    out["dz_actor"], out["grad_actor"] = g["dz"], g["grad"]
    return out


def value_step(value, state, min_q, *, log_prob=None, alpha=None, logged_action_uniform_prior=True,
               fp32=None):
    """rb200_ac_value_step (sac_trainer.py:329-343): V(s) against min_q, or
    min_q - alpha * clamp(log_prob) without the uniform prior.  `fp32`: "hidden_value".
    Returns loss, dz, hidden, grad."""
    s = _d(state)
    B = s.shape[0]
    tgt = _d(min_q).reshape(B)
    if not logged_action_uniform_prior:
        tgt = tgt - float(alpha) * _d(log_prob).reshape(B).clamp(LOG_PROB_MIN, LOG_PROB_MAX)
    net = Net64(value)
    v, zs, hs = net.forward(s, _get(fp32, "hidden_value"))
    d = v.reshape(B) - tgt
    loss = (d * d).mean()
    g = _grads(loss, [(net, zs)])[0]
    return {"loss": loss.detach(), "dz": g["dz"], "hidden": [h.detach() for h in hs],
            "grad": g["grad"], "value": v.detach().reshape(B)}
