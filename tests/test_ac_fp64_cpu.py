"""oracle/ac_fp64.py pinned to the fp32 restatements of the SAC / TD3 updates that the goldens
pin to the reference (td_oracle.sac_update / td3_update, per_ac_oracle, sac_value_oracle): one
update at a few small shapes, losses, TD targets, TD errors and every parameter gradient.  The
fp32 oracles carry their own rounding (atanh of a near-saturated fp32 action above all), so the
bound is fp32's, not the kernels' 1e-5."""
import math

import pytest
import torch

from oracle import ac_fp64 as X
from oracle import per_ac_oracle as P
from oracle import sac_value_oracle as V
from oracle import td_oracle as O

TOL32 = 2e-4   # fp32 autograd against float64


def _net(dims, acts, g, bias=0.3):
    n = O.make_net(dims, acts, g)
    for b in n["b"]:
        b.copy_(torch.randn(b.shape, generator=g) * bias)
    return n


def _batch(B, S, A, g):
    return {"state": torch.randn(B, S, generator=g), "action": torch.rand(B, A, generator=g) * 2 - 1,
            "next_state": torch.randn(B, S, generator=g), "reward": torch.randn(B, 1, generator=g),
            "not_terminal": (torch.rand(B, 1, generator=g) > 0.2).float()}


def _err(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _cmp_grads(g64, g32, what):
    flat = []
    for dW, db in g64:
        flat += [dW, db]
    assert len(flat) == len(g32), what
    for i, (a, b) in enumerate(zip(flat, g32)):
        assert _err(a, b) < TOL32, (what, i, _err(a, b))


CASES = [  # (B, S, A, sizes, acts, twin)
    (16, 5, 2, [32, 24], ["relu", "tanh"], True),
    (33, 7, 3, [40], ["leaky_relu"], False),
    (9, 3, 1, [17, 9, 13], ["softplus", "relu", "sigmoid"], True),
]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_sac_steps_match_fp32_oracle(case, weighted):
    B, S, A, sizes, acts, twin = CASES[case]
    g = torch.Generator().manual_seed(case)
    actor = _net([S] + sizes + [2 * A], acts + ["linear"], g)
    q1 = _net([S + A] + sizes + [1], acts + ["linear"], g)
    q2 = _net([S + A] + sizes + [1], acts + ["linear"], g) if twin else None
    batch = _batch(B, S, A, g)
    nn_, nc = torch.randn(B, A, generator=g), torch.randn(B, A, generator=g)
    w = torch.rand(B, generator=g) * 2 if weighted else None
    st = O.SacState(O.clone_net(actor), O.clone_net(q1), None if q2 is None else O.clone_net(q2),
                    lr=1e-3, entropy_temperature=0.1, learn_alpha=True, target_entropy=-float(A))
    log_alpha0, alpha0 = float(st.log_alpha.detach()), st.alpha
    ref = P.weighted_sac_update(st, batch, nn_, nc, w, gamma=0.9, tau=0.1)
    # critic step: the weights before the update (the targets are copies of the critics)
    got = X.critic_step(actor, q1, q2, q1, q2, batch, algo="sac", gamma=0.9, alpha=alpha0,
                        noise_next=nn_, sample_weight=w)
    assert _err(got["td_target"], ref["target"].reshape(-1)) < TOL32
    assert _err(got["loss"], ref["losses"][:2 if twin else 1]) < TOL32
    assert _err(got["q1_value"], ref["q1_value"]) < TOL32
    if weighted:
        assert _err(got["td_error"], ref["td_error"]) < TOL32
    _cmp_grads(got["grad_q1"], ref["grads"]["q1"], "q1")
    if twin:
        _cmp_grads(got["grad_q2"], ref["grads"]["q2"], "q2")
    # actor step: the critics after their Adam step, the actor and alpha before theirs
    ga = X.actor_step(actor, st.q1, st.q2, batch, algo="sac", alpha=alpha0, log_alpha=log_alpha0,
                      target_entropy=-float(A), noise_cur=nc)
    nl = 2 if twin else 1
    assert _err(ga["loss"], ref["losses"][nl]) < TOL32
    assert _err(ga["alpha_loss"], ref["losses"][nl + 1]) < TOL32
    assert _err(ga["alpha_grad"], ref["grads"]["alpha"][0]) < TOL32
    _cmp_grads(ga["grad_actor"], ref["grads"]["actor"], "actor")


@pytest.mark.parametrize("case", range(len(CASES)))
def test_td3_steps_match_fp32_oracle(case):
    B, S, A, sizes, acts, twin = CASES[case]
    g = torch.Generator().manual_seed(10 + case)
    actor = _net([S] + sizes + [A], acts + ["tanh"], g)
    q1 = _net([S + A] + sizes + [1], acts + ["linear"], g)
    q2 = _net([S + A] + sizes + [1], acts + ["linear"], g) if twin else None
    batch = _batch(B, S, A, g)
    # draws beyond the clip: noise_variance * n outside +-noise_clip on about half the rows
    nn_ = torch.randn(B, A, generator=g) * 4
    w = torch.rand(B, generator=g) * 2
    st = O.Td3State(O.clone_net(actor), O.clone_net(q1), None if q2 is None else O.clone_net(q2))
    ref = P.weighted_td3_update(st, batch, nn_, 0, w, gamma=0.9, tau=0.1, noise_variance=0.2,
                                noise_clip=0.5)
    got = X.critic_step(actor, q1, q2, q1, q2, batch, algo="td3", gamma=0.9, noise_next=nn_,
                        noise_variance=0.2, noise_clip=0.5, sample_weight=w)
    assert _err(got["td_target"], ref["target"].reshape(-1)) < TOL32
    assert _err(got["loss"], ref["losses"][:2 if twin else 1]) < TOL32
    assert _err(got["td_error"], ref["td_error"]) < TOL32
    _cmp_grads(got["grad_q1"], ref["grads"]["q1"], "q1")
    if twin:
        _cmp_grads(got["grad_q2"], ref["grads"]["q2"], "q2")
    ga = X.actor_step(actor, st.q1, st.q2, batch, algo="td3")
    assert _err(ga["loss"], ref["losses"][2 if twin else 1]) < TOL32
    _cmp_grads(ga["grad_actor"], ref["grads"]["actor"], "actor")


@pytest.mark.parametrize("crr", [None, {"indicator_fn_threshold": 0.1},
                                 {"exponent_beta": 0.5, "exponent_clamp": 2.0},
                                 {"exponent_beta": 2.0}])
@pytest.mark.parametrize("uniform_prior", [True, False])
def test_value_network_steps_match_fp32_oracle(crr, uniform_prior):
    B, S, A, sizes, acts = 21, 6, 2, [24, 16], ["relu", "tanh"]
    g = torch.Generator().manual_seed(7)
    actor = _net([S] + sizes + [2 * A], acts + ["linear"], g)
    q1 = _net([S + A] + sizes + [1], acts + ["linear"], g)
    q2 = _net([S + A] + sizes + [1], acts + ["linear"], g)
    value = _net([S] + sizes + [1], acts + ["linear"], g)
    batch = _batch(B, S, A, g)
    nc = torch.randn(B, A, generator=g)
    w = torch.rand(B, generator=g) * 2
    st = V.SacValueState(O.clone_net(actor), O.clone_net(q1), O.clone_net(q2), O.clone_net(value),
                         entropy_temperature=0.1, learn_alpha=True, target_entropy=-2.0,
                         logged_action_uniform_prior=uniform_prior, crr=crr)
    log_alpha0, alpha0 = float(st.log_alpha.detach()), st.alpha
    ref = V.sac_value_update(st, batch, nc, gamma=0.9, tau=0.1, sample_weight=w)
    got = X.critic_step(actor, q1, q2, None, None, batch, algo="sac", gamma=0.9, alpha=alpha0,
                        sample_weight=w, value_target=value)
    assert _err(got["td_target"], ref["target"].reshape(-1)) < TOL32
    assert _err(got["loss"], ref["losses"][:2]) < TOL32
    assert _err(got["td_error"], ref["td_error"]) < TOL32
    _cmp_grads(got["grad_q1"], ref["grads"]["q1"], "q1")
    _cmp_grads(got["grad_q2"], ref["grads"]["q2"], "q2")
    ga = X.actor_step(actor, st.q1, st.q2, batch, algo="sac", alpha=alpha0, log_alpha=log_alpha0,
                      target_entropy=-2.0, noise_cur=nc, value_net=value, crr=crr)
    assert _err(ga["loss"], ref["losses"][2]) < TOL32
    assert _err(ga["alpha_loss"], ref["losses"][3]) < TOL32
    _cmp_grads(ga["grad_actor"], ref["grads"]["actor"], "actor")
    # value step: the post-update alpha and the actor step's min_q / log-prob
    gv = X.value_step(value, batch["state"], ga["min_q"], log_prob=ga["log_prob"],
                      alpha=float(st.alpha), logged_action_uniform_prior=uniform_prior)
    assert _err(gv["loss"], ref["losses"][4]) < TOL32
    _cmp_grads(gv["grad"], ref["grads"]["value"], "value")


def test_fp32_bounds_and_saturated_log_prob():
    """The action bound is float32(1 - 1e-6); at it, the float64 log-prob of the fp32 action
    equals the fp32 oracle's (which squares the action in fp32) to fp32 precision."""
    assert X.ACT_HI == float(torch.tensor(1 - 1e-6, dtype=torch.float32))
    assert abs((1 - X.ACT_HI) / 1e-6 - 1.0132) < 1e-3
    g = torch.Generator().manual_seed(3)
    B, S, A = 12, 4, 3
    actor = _net([S, 8, 2 * A], ["relu", "linear"], g)
    actor["b"][-1][:A] = 20.0      # loc deep in tanh saturation
    actor["b"][-1][A:] = -8.0      # scale_log below the clamp
    s = torch.randn(B, S, generator=g)
    n = torch.randn(B, A, generator=g)
    a32, lp32 = O.gaussian_actor_forward(actor, s, n)
    assert (a32 == X.ACT_HI).all()
    out = X.Net64(actor).forward(X._d(s))[0]
    a_own, a, lp, _ = X.gaussian_head(out, n, fp32_action=a32)
    assert torch.equal(a_own, a32.double())
    assert _err(lp, lp32.reshape(-1)) < 1e-6
    assert (lp.detach() > X.LOG_PROB_MAX).all() or (lp.detach() < X.LOG_PROB_MIN).all()
    assert math.isfinite(float(lp.detach().sum()))
