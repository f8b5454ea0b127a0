"""rb200_crr_critic_head / rb200_crr_actor_head against their float64 references
(oracle/crr_oracle.py) at the edges of the shapes and value ranges they accept.  Arguments out of
range are refused by return code on the host, before any launch."""
import numpy as np
import pytest
import torch

from oracle import crr_oracle as CO
from tests import golden_util as G
from tests.kernel_util import _argmax_edge_rows

pytestmark = pytest.mark.gpu
TOL = 2e-5
RPB = 16  # rows per block


def _lib():
    from reagent_b200 import _lib

    return _lib


def _inputs(B, A, seed=0, noise_scale=None, prob=None):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    d = dict(actor_next=torch.tanh(r(B, A)), actor_out=torch.tanh(r(B, A)),
             q1t=r(B, A), q2t=r(B, A), q1=r(B, A), q2=r(B, A),
             action=torch.nn.functional.one_hot(torch.randint(A, (B,), generator=g), A).float(),
             reward=r(B), boost=r(A), nt=(torch.rand(B, generator=g) > 0.3).float(),
             prob=torch.rand(B, generator=g) * 0.8 + 0.1 if prob is None else prob,
             noise_next=None, noise=None)
    if noise_scale is not None:
        d["noise_next"], d["noise"] = r(B, A) * noise_scale, r(B, A) * noise_scale
    return d


def run_critic(d, twin=True, boost=True, gamma=0.9, batch=None, num_actions=None, check=True):
    L = _lib()
    B, A = d["q1"].shape
    dev = {k: None if v is None else v.cuda().contiguous() for k, v in d.items()}
    out = dict(y=torch.empty(B), s1=torch.empty(B), s2=torch.zeros(B), dz1=torch.empty(B, A),
               dz2=torch.zeros(B, A), parts=torch.zeros(2 * (-(-B // RPB))), loss=torch.zeros(2))
    out = {k: v.cuda() for k, v in out.items()}
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    a = L.CrrCriticArgsT()
    a.batch = B if batch is None else batch
    a.num_actions = A if num_actions is None else num_actions
    a.actor_next, a.noise_next = dev["actor_next"].data_ptr(), L.ptr(dev["noise_next"])
    a.q1_target_next, a.q1 = dev["q1t"].data_ptr(), dev["q1"].data_ptr()
    if twin:
        a.q2_target_next, a.q2 = dev["q2t"].data_ptr(), dev["q2"].data_ptr()
        a.q2_selected, a.dz_q2 = out["s2"].data_ptr(), out["dz2"].data_ptr()
    a.action, a.reward = dev["action"].data_ptr(), dev["reward"].data_ptr()
    a.reward_boost = dev["boost"].data_ptr() if boost else None
    a.not_terminal, a.gamma = dev["nt"].data_ptr(), gamma
    a.td_target, a.q1_selected, a.dz_q1 = (out["y"].data_ptr(), out["s1"].data_ptr(),
                                           out["dz1"].data_ptr())
    a.loss_partials, a.loss, a.tile_counter = (out["parts"].data_ptr(), out["loss"].data_ptr(),
                                               counter.data_ptr())
    rc = L.lib().rb200_crr_critic_head(a, L.cur_stream())
    if check:
        L.check(rc, "rb200_crr_critic_head")
        torch.cuda.synchronize()
        assert int(counter) == 0  # re-armed for the next launch
    return rc, {k: v.cpu() for k, v in out.items()}


def run_actor(d, *, beta=1.0, max_weight=20.0, entropy_coeff=0.0, clip_limit=10.0,
              activation="tanh", with_prob=True, with_dz=True, num_actions=None, check=True):
    L = _lib()
    B, A = d["q1"].shape
    dev = {k: None if v is None else v.cuda().contiguous() for k, v in d.items()}
    out = dict(w=torch.empty(B), dz=torch.empty(B, A), parts=torch.zeros(2 * (-(-B // RPB))),
               loss=torch.zeros(2))
    out = {k: v.cuda() for k, v in out.items()}
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    a = L.CrrActorArgsT()
    a.batch, a.num_actions = B, A if num_actions is None else num_actions
    a.actor_out, a.noise, a.q1 = dev["actor_out"].data_ptr(), L.ptr(dev["noise"]), dev["q1"].data_ptr()
    a.action = dev["action"].data_ptr()
    a.action_probability = dev["prob"].data_ptr() if with_prob else None
    a.inv_beta, a.max_weight, a.entropy_coeff, a.clip_limit = (1 / beta, max_weight,
                                                               entropy_coeff, clip_limit)
    a.action_activation = L.ACT[activation]
    a.weight = out["w"].data_ptr()
    a.dz = out["dz"].data_ptr() if with_dz else None
    a.loss_partials, a.loss, a.tile_counter = (out["parts"].data_ptr(), out["loss"].data_ptr(),
                                               counter.data_ptr())
    rc = L.lib().rb200_crr_actor_head(a, L.cur_stream())
    if check:
        L.check(rc, "rb200_crr_actor_head")
        torch.cuda.synchronize()
        assert int(counter) == 0
    return rc, {k: v.cpu() for k, v in out.items()}


def _close(got, ref, tol=TOL):
    assert G.rel_err(got, ref) < tol, G.rel_err(got, ref)


SHAPES = [(37, 2), (5, 3), (33, 31), (16, 32), (17, 33), (3, 1000), (2, 1024), (1, 4), (4096, 16)]


@pytest.mark.parametrize("B,A", SHAPES)
@pytest.mark.parametrize("twin", [True, False])
def test_critic_head_matches_fp64(B, A, twin):
    d = _inputs(B, A, seed=B + A, noise_scale=0.7 if A % 2 else None)
    _, o = run_critic(d, twin=twin)
    ref = CO.critic_head_fp64(d["actor_next"], d["noise_next"], d["q1t"], d["q2t"] if twin else None,
                              d["q1"], d["q2"] if twin else None, d["action"], d["reward"],
                              d["boost"], d["nt"], 0.9)
    _close(o["y"], ref["y"])
    _close(o["s1"], ref["q_sel"][0])
    _close(o["dz1"], ref["dz"][0])
    assert abs(float(o["loss"][0]) - ref["loss"][0]) <= TOL * max(1.0, ref["loss"][0])
    if twin:
        _close(o["s2"], ref["q_sel"][1])
        _close(o["dz2"], ref["dz"][1])
        assert abs(float(o["loss"][1]) - ref["loss"][1]) <= TOL * max(1.0, ref["loss"][1])
    else:
        assert float(o["loss"][1]) == 0.0
    # the gradient sits on the logged action only
    assert torch.equal(o["dz1"] != 0, (d["action"] != 0) & (o["dz1"] != 0))


@pytest.mark.parametrize("B,A", SHAPES)
@pytest.mark.parametrize("entropy_coeff", [0.0, 0.4])
def test_actor_head_matches_fp64(B, A, entropy_coeff):
    """The first rows log tied and NaN actions; the reference takes torch.argmax of them."""
    d = _inputs(B, A, seed=2 * B + A, noise_scale=0.7 if A % 2 else None)
    logged = _argmax_edge_rows(d["action"])
    d["action"] = torch.nn.functional.one_hot(logged.argmax(1), A).float()
    kw = dict(beta=0.7, max_weight=3.0, entropy_coeff=entropy_coeff, clip_limit=2.0)
    _, o = run_actor(dict(d, action=logged), **kw)
    _, o_onehot = run_actor(d, **kw)
    for k in o:
        assert torch.equal(o[k], o_onehot[k]), k
    ref = CO.actor_head_fp64(d["actor_out"], d["noise"], d["q1"], d["action"], d["prob"], **kw)
    _close(o["w"], ref["weight"])
    _close(o["dz"], ref["dz"])
    for i in range(2):
        assert abs(float(o["loss"][i]) - ref["loss"][i]) <= TOL * max(1.0, abs(ref["loss"][i]))
    if entropy_coeff == 0.0:
        assert float(o["loss"][0]) == float(o["loss"][1])


def test_shapes_out_of_range_are_refused_on_the_host():
    L = _lib()
    d = _inputs(4, 8)
    for bad in (dict(num_actions=1025), dict(num_actions=0), dict(batch=0)):
        rc, _ = run_critic(d, check=False, **bad)
        assert rc == -1, bad  # RB200_E_INVALID
    rc, _ = run_actor(d, num_actions=1025, check=False)
    assert rc == -1
    rc, _ = run_actor(d, entropy_coeff=0.1, with_prob=False, check=False)
    assert rc == -1 and b"action_probability" in L.lib().rb200_last_error()
    rc, _ = run_actor(d, entropy_coeff=0.0, with_prob=False, check=False)
    assert rc == 0
    torch.cuda.synchronize()


def test_weight_overflow_gives_max_weight_and_a_finite_loss():
    B, A = 24, 5
    d = _inputs(B, A, seed=3)
    a = d["action"].argmax(1)
    d["q1"] = torch.zeros(B, A)
    d["q1"][torch.arange(B), a] = torch.where(torch.arange(B) % 2 == 0, 400.0, -400.0)
    kw = dict(beta=0.5, max_weight=20.0)  # exp(800 * p) overflows fp32 on the even rows
    _, o = run_actor(d, **kw)
    assert torch.isfinite(o["loss"]).all() and torch.isfinite(o["dz"]).all()
    assert bool((o["w"][0::2] == 20.0).all()) and bool((o["w"][1::2] < 1e-30).all())
    ref = CO.actor_head_fp64(d["actor_out"], None, d["q1"], d["action"], d["prob"],
                             entropy_coeff=0.0, clip_limit=10.0, **kw)
    _close(o["w"], ref["weight"])
    _close(o["dz"], ref["dz"])


def test_ratio_clipped_low_high_and_not_at_all():
    B, A = 48, 4
    d = _inputs(B, A, seed=5)
    d["prob"] = torch.tensor([1e-3, 0.6, 1e6])[torch.arange(B) % 3]  # high clip, open, low clip
    kw = dict(beta=1.0, max_weight=20.0, entropy_coeff=0.5, clip_limit=1.5)
    _, o = run_actor(d, **kw)
    ref = CO.actor_head_fp64(d["actor_out"], None, d["q1"], d["action"], d["prob"], **kw)
    _close(o["dz"], ref["dz"])
    assert abs(float(o["loss"][1]) - ref["loss"][1]) <= TOL * max(1.0, abs(ref["loss"][1]))
    # through a clipped ratio no gradient flows: those rows have the gradient of
    # (-weight + entropy_coeff * ratio_constant) * log_pi alone
    l = d["actor_out"].double()
    p = torch.softmax(l, 1)
    onehot = d["action"].double()
    log_pi = (torch.log_softmax(l, 1) * onehot).sum(1)
    for rows, ratio in ((slice(0, None, 3), 1.5), (slice(2, None, 3), 1e-4)):
        coef = (-o["w"].double()[rows] + 0.5 * ratio) / B
        want = coef[:, None] * (onehot[rows] - p[rows]) * (1 - l[rows] ** 2)
        _close(o["dz"][rows], want)
    open_rows = slice(1, None, 3)
    raw = (p * onehot).sum(1) / d["prob"].double()
    assert bool(((raw[open_rows] > 1e-4) & (raw[open_rows] < 1.5)).all())
    coef = (-o["w"].double() + 0.5 * (raw + log_pi * raw))[open_rows] / B
    _close(o["dz"][open_rows], coef[:, None] * (onehot - p)[open_rows] * (1 - l[open_rows] ** 2))


def test_clamp_passes_the_gradient_exactly_at_plus_and_minus_one():
    B, A = 6, 4
    d = _inputs(B, A, seed=7)
    d["actor_out"] = torch.tensor([[0.5, 0.25, -0.5, 0.0]]).repeat(B, 1)
    # actor_out + noise = 1 exactly, -1 exactly, just outside on both sides
    d["noise"] = torch.tensor([[0.5, -1.25, -0.5 - 2 ** -20, 1.0 + 2 ** -20]]).repeat(B, 1)
    _, o = run_actor(d, activation="linear")
    ref = CO.actor_head_fp64(d["actor_out"], d["noise"], d["q1"], d["action"], d["prob"], beta=1.0,
                             max_weight=20.0, entropy_coeff=0.0, clip_limit=10.0,
                             activation="linear")
    _close(o["dz"], ref["dz"])
    assert bool((o["dz"][:, :2] != 0).all()) and bool((o["dz"][:, 2:] == 0).all())


@pytest.mark.parametrize("activation", ["linear", "tanh", "sigmoid", "leaky_relu"])
def test_every_action_activation_takes_the_same_route(activation):
    d = _inputs(19, 6, seed=9, noise_scale=0.3)
    if activation == "sigmoid":
        d["actor_out"] = torch.sigmoid(d["actor_out"] * 3)
    kw = dict(beta=1.0, max_weight=20.0, entropy_coeff=0.2, clip_limit=10.0)
    _, o = run_actor(d, activation=activation, **kw)
    ref = CO.actor_head_fp64(d["actor_out"], d["noise"], d["q1"], d["action"], d["prob"],
                             activation=activation, **kw)
    _close(o["dz"], ref["dz"])


def test_null_noise_equals_zero_noise_bit_for_bit():
    d = _inputs(45, 7, seed=11)
    z = dict(d, noise=torch.zeros(45, 7), noise_next=torch.zeros(45, 7))
    for run, kw in ((run_critic, {}), (run_actor, dict(entropy_coeff=0.3))):
        _, o0 = run(d, **kw)
        _, o1 = run(z, **kw)
        for k in o0:
            assert torch.equal(o0[k], o1[k]), (run.__name__, k)


def test_single_critic_equals_the_twin_heads_first_critic_bit_for_bit():
    d = _inputs(45, 7, seed=13, noise_scale=0.4)
    # the target differs (no min with q2), so compare with a q2 target that never wins the min
    d["q2t"] = d["q1t"] + 100.0
    _, tw = run_critic(d, twin=True)
    _, si = run_critic(d, twin=False)
    for k in ("y", "s1", "dz1"):
        assert torch.equal(tw[k], si[k]), k
    assert tw["loss"][0] == si["loss"][0]


def test_two_runs_are_bit_identical():
    d = _inputs(4099, 16, seed=15, noise_scale=0.2)
    for run, kw in ((run_critic, {}), (run_actor, dict(entropy_coeff=0.3))):
        _, o0 = run(d, **kw)
        _, o1 = run(d, **kw)
        for k in o0:
            assert torch.equal(o0[k], o1[k]), (run.__name__, k)


def test_actor_head_without_dz_computes_the_same_losses():
    d = _inputs(40, 5, seed=17)
    _, o0 = run_actor(d, entropy_coeff=0.3)
    _, o1 = run_actor(d, entropy_coeff=0.3, with_dz=False)
    assert torch.equal(o0["loss"], o1["loss"]) and torch.equal(o0["w"], o1["w"])
    assert np.isfinite(o1["loss"].numpy()).all()
