"""GPU parity of BehavioralCloningTrainer: the goldens of the unmodified reference through
train_step_gen and train_batch, a BCQ-imitator-sized update against the CPU oracle,
rb200_bc_xent_head alone at the edges of the shapes it accepts, the reference's own test, the
offline BC -> BCQ workflow, and the two-rank data-parallel update."""
import os

import pytest
import torch

from oracle import td_oracle as O
from tests import golden_util as G
from tests.builders import (CONFIG2_MAX_ADAM_OUTLIER_FRAC, CONFIG2_MAX_FLIPPED_ROWS, _free_port,
                            _record)
from tests.golden_cases import (BC_CASES, E2E, E2E_MAX_KEPT, E2E_MIN_BEHAVIOUR_KEPT, e2e_data,
                                e2e_metrics, golden_batch)
from tests.golden_util import TOL
from tests.kernel_util import _argmax_edge_rows

pytestmark = pytest.mark.gpu


def _rlt(b):
    from reagent_b200.core import types as rlt

    return rlt.BehavioralCloningModelInput(rlt.FeatureData(b["state"]), b["action"],
                                           b["possible_actions_mask"])


def _trainer(S, A, sizes, acts, lr, arrays=None, prefix="q0"):
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import BehavioralCloningTrainer

    net = FullyConnectedDQN(S, A, list(sizes), list(acts))
    if arrays is not None:
        G.load_into_module(arrays, prefix, net)
    return BehavioralCloningTrainer(net, optimizer=Optimizer__Union.default(lr=lr)).cuda()


def _close(got, want, tol=TOL):
    return abs(got - want) <= tol * max(1.0, abs(want))


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("name", BC_CASES)
def test_bc_matches_reference(name, fast):
    """Logits, loss, gradients and post-Adam parameters of every update, and validation_step."""
    arrays, meta = G.load(name)
    t = _trainer(meta["S"], meta["A"], meta["sizes"], meta["acts"], meta["lr"], arrays)
    opt = t.optimizers()[0]
    for it in range(meta["n_updates"]):
        b = golden_batch(arrays, f"batch{it}", "cuda")
        if fast:
            loss = float(t.train_batch(_rlt(b), it))
        else:
            out = t.training_step(_rlt(b), it, 0)
            assert out.grad_fn is not None
            opt.zero_grad()
            out.backward()
            opt.step()
            loss = float(out.detach())
        assert _close(loss, arrays["losses"][it]), (it, loss, arrays["losses"][it])
        want = torch.from_numpy(arrays[f"logits{it}"])
        mask = b["possible_actions_mask"].cpu().float()
        got = t._ws["scores"].cpu() + (-1e10) * (1 - mask)
        on = mask > 0
        assert G.rel_err(got[on], want[on]) < TOL
        assert torch.equal(got[~on], want[~on])  # x - 1e10 rounds to -1e10 for |x| < 512
        for i, g in enumerate(t.bc_net_grads()):
            assert G.rel_err(g, arrays[f"grad{it}.{i}"]) < TOL, (it, i)
        ps = list(t.bc_net.parameters())
        for i, (w, bb) in enumerate(G.net_pairs(arrays, f"q{it + 1}")):
            assert G.rel_err(ps[2 * i], w) < TOL, (it, i)
            assert G.rel_err(ps[2 * i + 1], bb) < TOL, (it, i)
    val = t.validation_step(_rlt(golden_batch(arrays, "val", "cuda")), 0)
    assert val.device.type == "cpu" and val.shape == ()
    assert _close(float(val), float(arrays["val_loss"])), (float(val), float(arrays["val_loss"]))


# ---------------------------------------------------------------------------
# BCQ-imitator size against the CPU oracle
# ---------------------------------------------------------------------------
def test_bc_imitator_sized_update_matches_oracle():
    """B 4096, S 128, FullyConnectedDQN(128, 16, [256, 128], relu), every action logged many
    times, random masks.  Loss and dz at 1e-5; a hidden unit within fp32 noise of 0 may take
    the other ReLU pattern, so gradients are compared in L2 / max norm and the number of such
    rows is bounded; post-Adam elements whose gradient is within noise of zero move by +-lr."""
    B, S, A, lr = 4096, 128, 16, 1e-3
    gen = torch.Generator().manual_seed(21)
    net = O.make_net([S, 256, 128, A], ["relu", "relu", "linear"], gen)
    for bb in net["b"]:
        bb.normal_(0, 0.1, generator=gen)
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = net["W"][i].numpy().copy(), net["b"][i].numpy().copy()
    labels = torch.randint(A, (B,), generator=gen)
    mask = (torch.rand(B, A, generator=gen) > 0.3).float()
    mask[torch.arange(B), labels] = 1.0
    b = dict(state=torch.randn(B, S, generator=gen),
             action=torch.nn.functional.one_hot(labels, A).float(), possible_actions_mask=mask)
    assert int(torch.bincount(labels, minlength=A).min()) > 100
    t = _trainer(S, A, [256, 128], ["relu", "relu"], lr, arrays)
    loss = float(t.train_batch(_rlt({k: v.cuda() for k, v in b.items()})))

    qo = O.clone_net(net, requires_grad=True)
    hs, x = [], b["state"]
    for w, bb, a in zip(qo["W"], qo["b"], qo["act"]):
        x = torch.nn.functional.linear(x, w, bb)
        if a == "relu":
            x = torch.relu(x)
            hs.append(x.detach())
    x.retain_grad()
    want_loss = torch.nn.functional.cross_entropy(x + (-1e10) * (1 - mask), labels)
    want_loss.backward()
    assert _close(loss, float(want_loss)), (loss, float(want_loss))
    net_ws = t._ws["net"]
    assert G.rel_err(net_ws.dz[-1], x.grad) < TOL
    same = torch.ones(B, dtype=torch.bool)
    for l in range(2):
        same &= ((net_ws.hidden[l].cpu() > 0) == (hs[l] > 0)).all(dim=1)
    flipped = int((~same).sum())
    assert flipped <= CONFIG2_MAX_FLIPPED_ROWS, flipped
    params = O.net_params(qo)
    grads = [p.grad.detach().clone() for p in params]
    l2mx = [G.grad_close(g, grads[i], f"grad {i}", l2_tol=1e-4, max_tol=1e-4)
            for i, g in enumerate(t.bc_net_grads())]
    O.AdamState(params, lr=lr).step(params, grads)
    fracs = []
    for i, p in enumerate(t.bc_net.parameters()):
        d = (p.detach().cpu().double() - params[i].detach().double()).abs()
        assert float(d.max()) <= 2.0 * lr * 1.01, i
        fracs.append(float((d > 1e-5 * float(params[i].abs().max())).double().mean()))
    _record("bc_imitator_sized", flipped_rows=flipped, grad_l2_rel=max(v[0] for v in l2mx),
            grad_max_rel=max(v[1] for v in l2mx), adam_outlier_frac=fracs)
    assert max(fracs) < CONFIG2_MAX_ADAM_OUTLIER_FRAC, fracs


# ---------------------------------------------------------------------------
# rb200_bc_xent_head alone
# ---------------------------------------------------------------------------
def _head(logits, labels, mask, with_dz=True):
    from reagent_b200 import _lib

    B, A = logits.shape
    dz = torch.full_like(logits, float("nan"))
    partials = torch.zeros(-(-B // _lib.BC_ROWS_PER_BLOCK), device="cuda")
    loss = torch.full((1,), float("nan"), device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    a = _lib.BcXentArgsT()
    a.batch, a.num_actions = B, A
    a.logits, a.labels, a.mask = logits.data_ptr(), labels.data_ptr(), mask.data_ptr()
    a.dz = dz.data_ptr() if with_dz else None
    a.loss_partials, a.loss, a.tile_counter = partials.data_ptr(), loss.data_ptr(), counter.data_ptr()
    _lib.check(_lib.lib().rb200_bc_xent_head(a, _lib.cur_stream()), "rb200_bc_xent_head")
    assert int(counter.item()) == 0  # reset for the next call (graph-capturable)
    return loss.cpu(), dz.cpu()


@pytest.mark.parametrize("A", [1, 2, 31, 32, 33, 1024])
def test_bc_xent_head_edges(A):
    """Against fp64 torch at B = 67 (not a multiple of the 8 rows per block): loss and dz,
    loss-only mode (dz untouched, same loss bits) and bit-identical repeats.  The first rows'
    labels have tied maxima or NaNs; the reference's label is their torch.argmax."""
    g = torch.Generator().manual_seed(A)
    B = 67
    x = torch.randn(B, A, generator=g) * 3
    y = torch.randint(A, (B,), generator=g)
    labels = _argmax_edge_rows(torch.nn.functional.one_hot(y, A).float())
    y = labels.argmax(1)
    mask = (torch.rand(B, A, generator=g) > 0.4).float()
    mask[torch.arange(B), y] = 1.0
    z = x.double() + (-1e10) * (1 - mask.double())
    want = torch.nn.functional.cross_entropy(z, y)
    want_dz = (torch.softmax(z, dim=1) - torch.nn.functional.one_hot(y, A).double()) / B
    xd, ld, md = x.cuda(), labels.cuda(), mask.cuda()
    loss, dz = _head(xd, ld, md)
    assert _close(float(loss), float(want), 1e-6), (float(loss), float(want))
    assert float((dz.double() - want_dz).abs().max()) <= 1e-6 * float(want_dz.abs().max()) + 1e-12
    loss_only, untouched = _head(xd, ld, md, with_dz=False)
    assert torch.equal(loss_only, loss) and bool(untouched.isnan().all())
    loss2, dz2 = _head(xd, ld, md)
    assert torch.equal(loss2, loss) and torch.equal(dz2, dz)
    if A == 1:
        assert float(loss) == 0.0 and bool((dz == 0).all())


# ---------------------------------------------------------------------------
# the reference's own test (reagent/test/training/test_behavioral_cloning.py)
# ---------------------------------------------------------------------------
def test_behavioral_cloning_v0():
    """200 batches x 4 epochs of the reference test's data through training.loop.run_update
    with the default Adam, then mean validation loss over 200 batches < 0.1 and softmax of the
    masked logits within 0.1 of the labels.  Seed 1, as the reference test's seed_everything(1)."""
    from oracle.make_bc_golden import _reference_test_batch
    from reagent_b200.core import types as rlt
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import BehavioralCloningTrainer, run_update

    torch.manual_seed(1)
    g = torch.Generator().manual_seed(1)

    def batches(n):
        return [_rlt({k: v.cuda() for k, v in _reference_test_batch(g).items()}) for _ in range(n)]

    train, evals = batches(200), batches(200)
    t = BehavioralCloningTrainer(FullyConnectedDQN(8, 4, [7, 6, 5], ["relu"] * 3),
                                 optimizer=Optimizer__Union.default()).cuda()
    for epoch in range(4):
        for i, b in enumerate(train):
            run_update(t, b, i)
    eval_loss = sum(float(t.validation_step(b, i)) for i, b in enumerate(evals)) / len(evals)
    assert abs(eval_loss) < 0.1, eval_loss
    b = evals[-1]
    probs = torch.softmax(t.bc_net(rlt.FeatureData(b.state.float_features), b.possible_actions_mask), dim=1)
    assert torch.allclose(b.action.double(), probs.double(), atol=1e-1)


# ---------------------------------------------------------------------------
# offline workflow: BC on logged data -> BCQ imitator of DQNTrainer
# ---------------------------------------------------------------------------
def test_offline_bc_then_bcq():
    """The scenario of test_bc_cpu.test_offline_bcq_scenario_on_the_oracle (same data, same
    initial weights, thresholds chosen there) with train_batch, then the trained network's
    `.fc` as the BCQ imitator: DQNTrainer's filtered next-action mask keeps the behaviour action
    on the held-out states."""
    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import DQNTrainer
    from reagent_b200.training.dqn_trainer import BCQConfig

    Wb, batches, held_out = e2e_data()
    S, A = E2E["S"], E2E["A"]
    net = O.make_net([S] + E2E["sizes"] + [A], ["relu", "relu", "linear"], torch.Generator().manual_seed(1))
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = net["W"][i].numpy(), net["b"][i].numpy()
    bc = _trainer(S, A, E2E["sizes"], ["relu", "relu"], E2E["lr"], arrays)
    for i, b in enumerate(batches):
        bc.train_batch(_rlt({k: v.cuda() for k, v in b.items()}), i)
    imitator = bc.bc_net.fc
    im_before = [p.detach().clone() for p in imitator.parameters()]

    torch.manual_seed(2)
    q = FullyConnectedDQN(S, A, [32], ["relu"])
    t = DQNTrainer(q, q.get_target_network(), actions=[str(i) for i in range(A)],
                   rl=RLParameters(gamma=0.9, target_update_rate=0.05), minibatch_size=len(held_out),
                   optimizer=Optimizer__Union.default(lr=1e-3),
                   evaluation=EvaluationParameters(calc_cpe_in_training=False),
                   imitator=imitator, bcq=BCQConfig(E2E["thr"])).cuda()
    gen = torch.Generator().manual_seed(3)
    B = len(held_out)
    act = torch.nn.functional.one_hot(torch.randint(A, (B,), generator=gen), A).float().cuda()
    batch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(torch.randn(B, S, generator=gen).cuda()),
        next_state=rlt.FeatureData(held_out.cuda()), reward=torch.randn(B, 1, generator=gen).cuda(),
        time_diff=None, step=None, not_terminal=torch.ones(B, 1).cuda(), action=act,
        next_action=act, possible_actions_mask=torch.ones(B, A).cuda(),
        possible_next_actions_mask=torch.ones(B, A).cuda(), extras=rlt.ExtraData())
    for it in range(3):
        t.train_batch(batch, it)
        kept_beh, kept = e2e_metrics(t.bcq_next_actions_mask.cpu(), Wb, held_out)
        _record("offline_bc_then_bcq", update=it, behaviour_kept=kept_beh, kept=kept)
        assert kept_beh >= E2E_MIN_BEHAVIOUR_KEPT, (it, kept_beh)
        assert kept <= E2E_MAX_KEPT, (it, kept)
    for p, p0 in zip(imitator.parameters(), im_before):
        assert torch.equal(p, p0)  # the imitator is frozen inside DQNTrainer


# ---------------------------------------------------------------------------
# N = 2 data parallel
# ---------------------------------------------------------------------------
def _dp_worker(rank, world, port, use_p2p, out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        from reagent_b200.training.data_parallel import enable_p2p, shard_rows

        if use_p2p:
            enable_p2p(dist.group.WORLD)
        B, S, A = 1024, 128, 16
        lo, hi = shard_rows(B, rank, world)
        g = torch.Generator(device=dev).manual_seed(3)
        state = torch.randn(B, S, device=dev, generator=g)
        act = torch.nn.functional.one_hot(torch.randint(A, (B,), device=dev, generator=g), A).float()
        mask = torch.ones(B, A, device=dev)

        def mk(sl):
            return _rlt(dict(state=state[sl], action=act[sl], possible_actions_mask=mask[sl]))

        trainers = []
        for _ in range(2):
            torch.manual_seed(11)
            trainers.append(_trainer(S, A, [256, 128], ["relu", "relu"], 1e-3))
        t_dp, t_full = trainers
        for it in range(2):
            t_full.train_batch(mk(slice(0, B)), it)
            t_dp.train_batch(mk(slice(lo, hi)), it, process_group=dist.group.WORLD)
        torch.cuda.synchronize()
        worst = frac = 0.0
        for a, b in zip(t_dp.parameters(), t_full.parameters()):
            scale = float(b.abs().max()) + 1e-30
            d = (a.detach().double() - b.detach().double()).abs()
            worst = max(worst, float(d.max()) / scale)
            frac = max(frac, float((d > 1e-5 * scale).double().mean()))
        flat = torch.cat([p.detach().reshape(-1) for p in t_dp.parameters()])
        other = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(other, flat)
        out.put((rank, worst, frac, all(torch.equal(o, flat) for o in other)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_p2p", [True, False])
def test_bc_two_rank_update_matches_full_batch(use_p2p):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, use_p2p, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(500)
        assert p.exitcode == 0, f"worker exit code {p.exitcode}"
    for rank, worst, frac, same in [out.get(timeout=10) for _ in range(2)]:
        # as test_dp_gpu: +-lr moves of elements whose gradient is within noise of zero
        assert worst < 0.05, (rank, worst)
        assert frac < 2e-3, (rank, frac)
        assert same, "ranks diverged"
