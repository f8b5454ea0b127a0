"""GPU parity of batch-constrained Q-learning: DQNTrainer(imitator=, bcq=) and
BatchConstrainedDQN against golden vectors of the unmodified reference, the config-2-sized
update against the CPU oracle, rb200_bcq_filter at the edges of the shapes it accepts, and the
captured FusedDqnStep against the eager update."""
import math
import random

import numpy as np
import pytest
import torch

from oracle import bcq_oracle as BO
from oracle import td_oracle as O
from tests import golden_util as G
from tests.builders import (K2_PATHS, _assert_k2, _build_bcq, _golden_batch, _record, _rlt_batch,
                            _select_k2)
from tests.golden_cases import BCQ_DQN_CASES
from tests.golden_util import TOL

pytestmark = pytest.mark.gpu


def _close(got, want):
    return abs(got - want) <= TOL * max(1.0, abs(want))


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("path", K2_PATHS)
@pytest.mark.parametrize("name", BCQ_DQN_CASES)
def test_bcq_dqn_matches_reference(name, path, fast, monkeypatch):
    """Generator path (training_step per optimizer) and train_batch, on both K2 kernels: the
    filtered next-action mask bit for bit, losses / CPE losses / first-update gradients / final
    parameters at 1e-5, and the caller's batch masks untouched."""
    from reagent_b200.training.workspace import param_grads

    _select_k2(monkeypatch, path)
    arrays, meta = G.load(name)
    cpe = meta["cpe_metrics"] is not None
    t = _build_bcq(meta, arrays)
    b, batch = _golden_batch(arrays, meta)
    masks_before = (b["possible_next_actions_mask"].clone(), b["possible_actions_mask"].clone())
    opts = t.optimizers()
    assert len(opts) == (4 if cpe else 2)

    def check_first_update():
        assert torch.equal(t.bcq_next_actions_mask.cpu(), torch.from_numpy(arrays["bcq.next_mask0"]))
        for i, g in enumerate(t.q_network_grads()):
            assert G.rel_err(g, arrays[f"grad0.{i}"]) < TOL, f"grad {i}"
        assert G.rel_err(t.all_action_scores, arrays["all_q0"]) < TOL
        if cpe:
            for net, key in ((t.reward_network, "grad0r"), (t.q_network_cpe, "grad0c")):
                for i, g in enumerate(param_grads(net.arena, list(net.parameters()))):
                    assert G.rel_err(g, arrays[f"{key}.{i}"]) < TOL, (key, i)

    for it in range(meta["n_updates"]):
        if fast:
            losses = [float(t.train_batch(batch, it))]
            if cpe:
                losses += [float(x) for x in t.cpe_losses]
            if it == 0:
                check_first_update()
        else:
            losses = []
            for i, opt in enumerate(opts):
                loss = t.training_step(batch, it, i)
                if it == 0 and i == (1 if cpe else 0):
                    check_first_update()  # CPE gradients exist from the first CPE yield on
                opt.zero_grad()
                loss.backward()
                opt.step()
                losses.append(float(loss))
            losses = losses[:-1]  # the soft update's
        want = [arrays["losses"][it]] + (list(arrays["cpe_losses"][it]) if cpe else [])
        assert all(_close(g, w) for g, w in zip(losses, want)), (it, losses, want)
    _assert_k2(t, path)
    nets = [(t.q_network, "qN"), (t.q_network_target, "qtN")]
    if cpe:
        nets += [(t.reward_network, "rN"), (t.q_network_cpe, "cN"), (t.q_network_cpe_target, "ctN")]
    for net, prefix in nets:
        ps = list(net.parameters())
        for i, (w, bb) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < TOL, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], bb) < TOL, (prefix, i)
    # the trainer never writes the caller's tensors (the reference's `*=` does)
    assert torch.equal(b["possible_next_actions_mask"], masks_before[0])
    assert torch.equal(b["possible_actions_mask"], masks_before[1])
    # and the imitator is frozen
    for i, (w, bb) in enumerate(G.net_pairs(arrays, "im")):
        assert torch.equal(t.bcq_imitator.dnn[i][0].weight.cpu(), torch.from_numpy(w))


def test_bcq_compute_td_loss_only_uses_the_filter():
    """validation_step's loss (compute_td_loss_only) filters like the training step."""
    arrays, meta = G.load("dqn_bcq_huber_double")
    t = _build_bcq(meta, arrays)
    _, batch = _golden_batch(arrays, meta)
    loss = float(t.compute_td_loss_only(batch))
    assert torch.equal(t.bcq_next_actions_mask.cpu(), torch.from_numpy(arrays["bcq.next_mask0"]))
    assert _close(loss, arrays["losses"][0]), (loss, arrays["losses"][0])


def _load_model(arrays, meta):
    from reagent_b200.models import BatchConstrainedDQN, FullyConnectedDQN, FullyConnectedNetwork

    q = FullyConnectedDQN(meta["S"], meta["A"], meta["sizes"], ["relu"] * len(meta["sizes"]))
    im = FullyConnectedNetwork([meta["S"]] + meta["imitator_sizes"] + [meta["A"]],
                               meta["imitator_acts"])
    G.load_into_module(arrays, "q0", q)
    G.load_into_module(arrays, "im", im)
    return BatchConstrainedDQN(meta["S"], q, im, meta["thr"]).cuda()


def test_batch_constrained_dqn_forward_matches_reference():
    from reagent_b200.core import types as rlt
    from reagent_b200.gym.policies import GreedyActionSampler, Policy, discrete_dqn_scorer

    arrays, meta = G.load("bcq_model_forward")
    m = _load_model(arrays, meta)
    x = rlt.FeatureData(torch.from_numpy(arrays["state"]).cuda())
    out = m(x).cpu()
    want = torch.from_numpy(arrays["out"])
    dropped = torch.from_numpy(arrays["r"] < meta["thr"])
    assert 0 < int(dropped.sum()) < dropped.numel()
    assert torch.equal(out[dropped], want[dropped])  # q + (-1e10): exact
    assert G.rel_err(out[~dropped], want[~dropped]) < TOL
    # act time: the scorer composes with the model, greedy never picks a dropped action
    scorer = discrete_dqn_scorer(m)
    scores = scorer(x)
    assert torch.equal(scores.cpu(), out)
    act = Policy(scorer, GreedyActionSampler()).act(x)
    picked = act.action.argmax(dim=1)
    assert not bool(dropped[torch.arange(len(picked)), picked].any())


# ---------------------------------------------------------------------------
# config-2 size against the CPU oracle
# ---------------------------------------------------------------------------
# The imitator's logits come from the fused MLP forward (3xTF32 products): a mask entry whose
# oracle filter value r lies closer to the threshold than that forward's error can reach (r =
# exp(x - max x), so |d log r| <= 2 max |d x|) may flip, and that is not a parity question.
# Those entries are excluded from the bit-for-bit comparison and their number is bounded.
CONFIG2_MAX_NEAR_THRESHOLD_FRAC = 1e-3


@pytest.mark.parametrize("path", K2_PATHS)
def test_bcq_config2_matches_oracle(path, monkeypatch):
    """B 4096, S 128, A 16, q [256,128], imitator [128,256,128,16] (relu), threshold 0.3."""
    from reagent_b200.models import FullyConnectedNetwork

    _select_k2(monkeypatch, path)
    B, S, A, thr = 4096, 128, 16, 0.3
    meta = dict(S=S, A=A, B=B, sizes=[256, 128], acts=["relu", "relu"], gamma=0.99, tau=0.005,
                loss="huber", maxq=True, multi_steps=None, time_diff=False, boost=None,
                double_q=True, lr=1e-3, bcq=thr)
    gen = torch.Generator().manual_seed(5)
    q = O.make_net([S, 256, 128, A], ["relu", "relu", "linear"], gen)
    qt = O.clone_net(q)
    for w in qt["W"]:
        w.add_(torch.randn(w.shape, generator=gen) * 0.02)
    im = O.make_net([S, 256, 128, A], ["relu", "relu", "linear"], gen)  # drops ~2/3 of the actions
    arrays = {}
    for prefix, net in (("q0", q), ("qt0", qt), ("im", im)):
        for i in range(3):
            arrays[f"{prefix}.W{i}"] = net["W"][i].numpy().copy()
            arrays[f"{prefix}.b{i}"] = net["b"][i].numpy().copy()
    act = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.005).float()
    pnam = (torch.rand(B, A, generator=gen) > 0.2).float()
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen), time_diff=torch.ones(B, 1), step=None,
             not_terminal=nt, action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=pnam)
    imitator = FullyConnectedNetwork([S, 256, 128, A], ["relu", "relu", "linear"])
    t = _build_bcq(meta, arrays, imitator=imitator)
    batch = _rlt_batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    loss = float(t.compute_td_loss_only(batch))
    _assert_k2(t, path)
    keep, r = BO.bcq_filter(im, b["next_state"], thr)
    oracle_mask = pnam * keep
    gpu_mask = t.bcq_next_actions_mask.cpu()
    logits_ref = O.mlp(im, b["next_state"])
    logits = t._ws["bcq_logits"].cpu()
    assert G.rel_err(logits, logits_ref) < TOL
    band = 2.0 * float((logits.double() - logits_ref.double()).abs().max()) + 1e-6
    near = (r.double().log() - math.log(thr)).abs() <= band
    drop_frac = float((keep == 0).double().mean())
    assert 0.1 < drop_frac < 0.9, drop_frac
    n_near, n_near_1e5 = int(near.sum()), int(((r.double() - thr).abs() <= 1e-5 * thr).sum())
    flipped = int((gpu_mask != oracle_mask).sum())
    _record("bcq_config2", path=path, log_r_band=band, near_threshold=n_near,
            near_threshold_1e5_rel=n_near_1e5, flipped=flipped, dropped=drop_frac)
    assert n_near <= CONFIG2_MAX_NEAR_THRESHOLD_FRAC * near.numel(), n_near
    assert torch.equal(gpu_mask[~near], oracle_mask[~near])
    rows = (gpu_mask == oracle_mask).all(dim=1)
    kw = dict(gamma=meta["gamma"], double_q=True, maxq=True, loss="huber")
    lo, aux = BO.dqn_td_loss(q, qt, b, imitator=im, bcq_threshold=thr, **kw)
    assert G.rel_err(t._ws["td_target"].cpu()[rows], aux["target"].reshape(-1)[rows]) < TOL
    if bool(rows.all()):
        assert _close(loss, float(lo)), (loss, float(lo))
    else:  # the loss over every row, with the GPU's mask on the rows whose entries flipped
        bg = dict(b, possible_next_actions_mask=gpu_mask)
        lg, _ = O.dqn_td_loss(q, qt, bg, **kw)
        assert _close(loss, float(lg)), (loss, float(lg))


# ---------------------------------------------------------------------------
# rb200_bcq_filter alone
# ---------------------------------------------------------------------------
def _filter(logits, thr, mask_in=None, q_in=None):
    from reagent_b200 import _lib

    B, A = logits.shape
    out = torch.full_like(logits, float("nan"))
    trainer = q_in is None
    rc = _lib.lib().rb200_bcq_filter(
        logits.data_ptr(), B, A, float(thr), None if mask_in is None else mask_in.data_ptr(),
        out.data_ptr() if trainer else None, None if trainer else q_in.data_ptr(),
        None if trainer else out.data_ptr(), _lib.cur_stream())
    _lib.check(rc, "rb200_bcq_filter")
    return out.cpu()


@pytest.mark.parametrize("A", [1, 2, 31, 32, 33, 1024])
def test_bcq_filter_kernel_edges(A):
    """Against an fp64 torch computation: thresholds 0 (keep all), 1 (keep only ties with the
    max) and 0.3, with tied maxima, both output modes, with and without an input mask."""
    g = torch.Generator().manual_seed(A)
    B = 67
    # logits on a 0.25 grid: distinct values differ by far more than fp32 noise in r
    x = torch.randint(-24, 8, (B, A), generator=g).float() * 0.25
    x[:, 0] = x.max(dim=1).values            # a tie with the row maximum in every row (A > 1)
    x[B - 1] = 1.5                           # a row of equal logits
    xd = x.cuda()
    p = torch.softmax(x.double(), dim=1)
    r = p / p.max(dim=1, keepdim=True).values
    mask = (torch.rand(B, A, generator=g) > 0.3).float()
    q = torch.randn(B, A, generator=g) * 10
    for thr in (0.0, 1.0, 0.3):
        keep = (r >= thr).float()
        exact = (r - thr).abs() > 1e-5 * max(thr, 1e-30)
        if thr == 1.0:
            keep = (x == x.max(dim=1, keepdim=True).values).float()
            exact = torch.ones_like(exact)
        if thr == 0.0:
            exact = torch.ones_like(exact)
        got = _filter(xd, thr)
        assert torch.equal(got[exact], keep[exact]), thr
        assert torch.equal(_filter(xd, thr, mask_in=mask.cuda())[exact], (mask * keep)[exact])
        gq = _filter(xd, thr, q_in=q.cuda())
        want_q = q + (-1e10) * (1.0 - got)  # float32 arithmetic of the reference's penalty
        assert torch.equal(gq, want_q), thr
    assert torch.equal(_filter(xd, 1.0)[:, 0], torch.ones(B))
    assert torch.equal(_filter(xd, 1.0)[B - 1], torch.ones(A))


# ---------------------------------------------------------------------------
# FusedDqnStep (the whole update as one CUDA graph) with BCQ
# ---------------------------------------------------------------------------
FS, FA, FB, FCAP = 24, 5, 256, 4096


def _fused_setup(prioritized=True):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import FullyConnectedDQN, FullyConnectedNetwork
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, ReplayBuffer
    from reagent_b200.training import DQNTrainer
    from reagent_b200.training.dqn_trainer import BCQConfig

    dev = torch.device("cuda", 0)
    rng = np.random.RandomState(3)
    n = FCAP - 7
    data = dict(observation=rng.standard_normal((n, FS)).astype(np.float32),
                action=rng.randint(0, FA, n).astype(np.int64),
                reward=rng.standard_normal(n).astype(np.float32),
                terminal=rng.rand(n) < 0.02, priority=rng.uniform(0.1, 10.0, n))
    if prioritized:
        rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=FCAP, batch_size=FB, device=dev)
    else:
        rb = ReplayBuffer(stack_size=1, replay_capacity=FCAP, batch_size=FB, device=dev)
        data.pop("priority")
    rb.add_batch(**data)
    torch.manual_seed(1)
    q = FullyConnectedDQN(FS, FA, [48, 32], ["relu", "relu"])
    im = FullyConnectedNetwork([FS, 32, FA], ["relu", "linear"])
    with torch.no_grad():
        im.dnn[-1][0].weight.mul_(4.0)
    t = DQNTrainer(q, q.get_target_network(), actions=[str(i) for i in range(FA)],
                   rl=RLParameters(gamma=0.9, target_update_rate=0.05, q_network_loss="huber"),
                   double_q_learning=True, minibatch_size=FB,
                   optimizer=Optimizer__Union.default(lr=1e-2),
                   evaluation=EvaluationParameters(calc_cpe_in_training=False),
                   imitator=im, bcq=BCQConfig(0.3)).to(dev)
    return rb, t


def _seed():
    random.seed(7)
    torch.manual_seed(7)
    np.random.seed(7)


def _same_params(t, t2):
    for a, b in zip(t.q_network.parameters(), t2.q_network.parameters()):
        assert torch.equal(a, b)
    for a, b in zip(t.q_network_target.parameters(), t2.q_network_target.parameters()):
        assert torch.equal(a, b)


def _donor():
    from reagent_b200.models import FullyConnectedNetwork

    torch.manual_seed(99)
    d = FullyConnectedNetwork([FS, 32, FA], ["relu", "linear"])
    with torch.no_grad():
        d.dnn[-1][0].weight.mul_(6.0)
    return d.state_dict()


@pytest.mark.parametrize("prefetch", [False, True])
def test_bcq_fused_step_matches_eager(prefetch):
    """Host random stream, with a load_state_dict on the imitator between two replays: the
    captured imitator forward reads the arena in place, so the new weights take effect."""
    from reagent_b200.training.fused_step import FusedDqnStep

    n, swap, donor = 7, 4, _donor()
    rb, t = _fused_setup()
    _seed()
    eager, masks = [], []
    for i in range(n + 1):  # FusedDqnStep's constructor runs one warm-up update
        if i == swap:
            t.bcq_imitator.load_state_dict(donor)
        eager.append(float(t.train_batch(rb.sample_discrete_dqn_batch(FB, FA))))
        masks.append(t.bcq_next_actions_mask.clone())
    rb2, t2 = _fused_setup()
    _seed()
    fused = FusedDqnStep(t2, rb2, FB, prefetch=prefetch)
    got = []
    for i in range(1, n + 1):
        if i == swap:
            t2.bcq_imitator.load_state_dict(donor)
        lh = fused.step()
        torch.cuda.synchronize()
        got.append(float(lh[0]))
        if not prefetch:
            assert torch.equal(t2.bcq_next_actions_mask, masks[i])
    assert got == eager[1:], (got, eager[1:])
    _same_params(t, t2)


@pytest.mark.parametrize("online", [False, True])
def test_bcq_fused_step_device_rng_matches_eager(online):
    """rng="device" (and online=True: one transition added per step): the captured update
    against the same device-resident draws run eagerly."""
    from reagent_b200.replay_memory.device_replay import DeviceReplay
    from reagent_b200.training.fused_step import FusedDqnStep

    rng = np.random.RandomState(11)
    extra = dict(observation=rng.standard_normal((8, FS)).astype(np.float32),
                 action=rng.randint(0, FA, 8).astype(np.int64),
                 reward=rng.standard_normal(8).astype(np.float32),
                 terminal=np.zeros(8, bool), priority=rng.uniform(0.1, 10.0, 8))
    rb, t = _fused_setup()
    _seed()
    dr = DeviceReplay(rb, stage_rows=1, stage_slots=2)
    eager = []
    for i in range(7):
        if online and i > 0:  # the constructor's warm-up update adds nothing
            dr.add(**{k: v[i] for k, v in extra.items()})
        idx = dr.draw_indices(FB)
        eager.append(float(t.train_batch(rb.sample_discrete_dqn_batch(FB, FA, indices=idx))))
    rb2, t2 = _fused_setup()
    _seed()
    fused = FusedDqnStep(t2, rb2, FB, rng="device", online=online)
    got = []
    for i in range(1, 7):
        lh = fused.step({k: v[i] for k, v in extra.items()} if online else None)
        torch.cuda.synchronize()
        got.append(float(lh[0]))
    assert got == eager[1:], (got, eager[1:])
    _same_params(t, t2)
