"""rb200_pg_head alone against the fp64 reference of oracle/pg_oracle.py, at A = 1, 33 and 1024
(one column per lane, two, and 32), with masks, rows of several trajectories, the off-policy
REINFORCE clip, PPO ratios on both sides of the clip and with the entropy bonus, the value
baseline, a PPO ratio exactly at both clip bounds, where torch.minimum ties and torch.clamp's
closed interval pass the full gradient, and logged actions with tied maxima or NaNs, read as
torch.argmax reads them."""
import math

import pytest
import torch

from oracle import pg_oracle as PO
from tests import golden_util as G
from tests.kernel_util import _argmax_edge_rows

pytestmark = pytest.mark.gpu

LENGTHS = [1, 17, 22]


def _launch(scores, action, *, mask=None, loss_kind, returns, value=None, logged=None,
            temperature=1.0, ppo_epsilon=0.2, entropy_weight=0.0, log_clip_param=0.0,
            value_scale=1.0, lengths=LENGTHS):
    from reagent_b200 import _lib

    dev = torch.device("cuda")
    R, A = scores.shape
    t = {k: (None if v is None else v.float().to(dev).contiguous()) for k, v in dict(
        scores=scores, action=action, mask=mask, returns=returns, value=value,
        logged=logged).items()}
    offs = torch.tensor(PO.pack_offsets(lengths), dtype=torch.int32, device=dev)
    dz = torch.full((R, A), float("nan"), device=dev)
    dz_value = torch.full((R,), float("nan"), device=dev)
    adv = torch.full((R,), float("nan"), device=dev)
    partials = torch.zeros(2 * -(-R // _lib.PG_ROWS_PER_BLOCK), device=dev)
    loss = torch.zeros(2, device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    a = _lib.PgHeadArgsT()
    a.rows, a.num_actions, a.n_traj, a.offsets = R, A, len(lengths), offs.data_ptr()
    a.scores, a.action, a.mask = t["scores"].data_ptr(), t["action"].data_ptr(), _lib.ptr(t["mask"])
    a.logged_log_prob, a.returns, a.value = _lib.ptr(t["logged"]), _lib.ptr(t["returns"]), _lib.ptr(t["value"])
    a.temperature, a.reward_clip = temperature, 1e6
    a.log_clip_param, a.entropy_weight = log_clip_param, entropy_weight
    a.ppo_clip_lo, a.ppo_clip_hi = 1.0 - ppo_epsilon, 1.0 + ppo_epsilon
    a.value_scale, a.loss_kind = value_scale, loss_kind
    a.advantage_kind = _lib.PG_ADV_RETURNS if value is None else _lib.PG_ADV_BASELINE
    a.advantage_out, a.dz = adv.data_ptr(), dz.data_ptr()
    a.dz_value = dz_value.data_ptr() if value is not None else None
    a.loss_partials, a.loss, a.tile_counter = partials.data_ptr(), loss.data_ptr(), counter.data_ptr()
    _lib.check(_lib.lib().rb200_pg_head(a, _lib.cur_stream()), "rb200_pg_head")
    return loss.cpu(), dz.cpu(), dz_value.cpu(), adv.cpu()


def _inputs(A, seed):
    g = torch.Generator().manual_seed(seed)
    R = sum(LENGTHS)
    scores = torch.randn(R, A, generator=g) * 2
    act = torch.randint(A, (R,), generator=g)
    action = _argmax_edge_rows(torch.nn.functional.one_hot(act, A).float())
    act = action.argmax(1)  # the reference's logged action, which the head must pick too
    mask = (torch.rand(R, A, generator=g) > 0.3).float()
    mask[torch.arange(R), act] = 1.0
    returns = torch.randn(R, generator=g)
    return g, scores, action, mask, returns


def _lp64(scores, mask, action, temperature):
    z = PO.logits(scores.double(), mask.double(), temperature)
    return torch.log_softmax(z, 1).gather(1, action.argmax(1, keepdim=True)).squeeze(1)


@pytest.mark.parametrize("A", [1, 33, 1024])
def test_reinforce_head_matches_fp64(A):
    from reagent_b200 import _lib

    g, scores, action, mask, returns = _inputs(A, A)
    for off_policy in (False, True):
        logged = None
        if off_policy:  # ratios on both sides of clip_param = 1.5
            logged = (_lp64(scores, mask, action, 0.7) + torch.randn(len(returns), generator=g)).float()
        loss, dz, _, adv = _launch(scores, action, mask=mask, loss_kind=_lib.PG_LOSS_REINFORCE,
                                   returns=returns, logged=logged, temperature=0.7,
                                   log_clip_param=math.log(1.5))
        want_loss, want_dz = PO.head_fp64(scores, mask, action, returns, temperature=0.7,
                                          ppo=False, logged=logged, clip_param=1.5)
        assert torch.equal(adv, returns)
        assert abs(float(loss[0]) - want_loss) <= 1e-5 * max(1.0, abs(want_loss))
        assert G.rel_err(dz, want_dz) < 1e-5
        if A > 1:
            assert float(dz.abs().max()) > 0


@pytest.mark.parametrize("A", [1, 33, 1024])
def test_ppo_head_matches_fp64_with_entropy_and_a_value_baseline(A):
    from reagent_b200 import _lib

    g, scores, action, mask, returns = _inputs(A, 100 + A)
    R = len(returns)
    logged = (_lp64(scores, mask, action, 1.3) + 0.5 * torch.randn(R, generator=g)).float()
    value = torch.randn(R, generator=g)
    loss, dz, dz_value, adv = _launch(scores, action, mask=mask, loss_kind=_lib.PG_LOSS_PPO,
                                      returns=returns, value=value, logged=logged,
                                      temperature=1.3, entropy_weight=0.05)
    adv64 = returns.double() - value.double()
    want_loss, want_dz = PO.head_fp64(scores, mask, action, adv64, temperature=1.3, ppo=True,
                                      logged=logged, ppo_epsilon=0.2, entropy_weight=0.05)
    assert G.rel_err(adv, adv64) < 1e-6
    assert abs(float(loss[0]) - want_loss) <= 1e-5 * max(1.0, abs(want_loss))
    assert G.rel_err(dz, want_dz) < 1e-5
    assert G.rel_err(dz_value, 2.0 * (value.double() - returns.double())) < 1e-6
    want_v = float(((value.double() - returns.double()) ** 2).sum())
    assert abs(float(loss[1]) - want_v) <= 1e-5 * want_v
    rho = torch.exp(_lp64(scores, mask, action, 1.3) - logged.double())
    if A > 1:
        assert bool((rho < 0.8).any()) and bool((rho > 1.2).any())


@pytest.mark.parametrize("A", [2, 33, 1024])
def test_ppo_ratio_on_both_clip_bounds_passes_the_full_gradient(A):
    """logged = the kernel's own log pi (read back one row at a time from REINFORCE's loss,
    -log pi for a return of 1), so rho = exp(0) = 1 exactly, and epsilon 0 puts both clip
    bounds on it: the two sides of torch.minimum tie and the clamp passes, so the gradient is
    REINFORCE's, bit for bit, and the fp64 reference's."""
    from reagent_b200 import _lib

    g, scores, action, mask, returns = _inputs(A, 200 + A)
    R = len(returns)
    lp = torch.empty(R)
    for r in range(R):
        one = _launch(scores[r:r + 1], action[r:r + 1], mask=mask[r:r + 1],
                      loss_kind=_lib.PG_LOSS_REINFORCE, returns=torch.ones(1), lengths=[1])[0]
        lp[r] = -one[0]
    loss, dz, _, _ = _launch(scores, action, mask=mask, loss_kind=_lib.PG_LOSS_PPO,
                             returns=returns, logged=lp, ppo_epsilon=0.0)
    _, dz_reinforce, _, _ = _launch(scores, action, mask=mask, loss_kind=_lib.PG_LOSS_REINFORCE,
                                    returns=returns)
    assert torch.equal(dz, dz_reinforce)
    assert float(dz.abs().max()) > 0
    # fp64: its own log pi as the logged one, so its rho is exactly 1 too
    want_loss, want_dz = PO.head_fp64(scores, mask, action, returns, temperature=1.0, ppo=True,
                                      logged=_lp64(scores, mask, action, 1.0), ppo_epsilon=0.0)
    assert G.rel_err(dz, want_dz) < 1e-5
    assert abs(float(loss[0]) - want_loss) <= 1e-5 * max(1.0, abs(want_loss))
