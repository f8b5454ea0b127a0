"""Pins the summation order of every loss kernel's deterministic mean bit for bit.

Each loss kernel writes its per-block partials to loss_partials, and the last block to finish
reduces them in one of two fixed orders (rb200_common.cuh, DESIGN.md section 3):
  serial -- one thread adds the partials in block order (dqn_td_rows_kernel, dqn_td_tc_kernel,
            pdqn_head_kernel, cpe_heads_kernel, ac_critic_rows_kernel, ac_actor_rows_kernel);
  block  -- thread t of the last block adds partials t, t + 256, ..., each warp reduces with an
            xor butterfly, and thread 0 adds the warp sums in order (c51_head_kernel,
            qr_head_kernel, bc_xent_head_kernel).
Each test runs one kernel once, reads back the partials it wrote, and requires the loss bits to
equal a float32 restatement of that kernel's order and final arithmetic."""

import numpy as np
import pytest
import torch

from reagent_b200 import _lib
from tests.builders import _assert_k2, _build_trainer, _pbatch, _rlt_batch, _select_k2
from tests.kernel_util import _call, _set_ws, _ws

pytestmark = pytest.mark.gpu
f32 = np.float32


def _serial(p, n, ch=1):
    tot = [f32(0)] * ch
    for i in range(n):
        for c in range(ch):
            tot[c] = f32(tot[c] + p[ch * i + c])
    return tot


def _block(p, n, w=None, threads=256):
    vals = p[:n] if w is None else p[:n] * w[:n]   # float32 products: __fmul_rn
    lanes = np.zeros(threads, f32)
    for t in range(threads):
        s = f32(0)
        for i in range(t, n, threads):
            s = f32(s + vals[i])
        lanes[t] = s
    v = lanes.reshape(threads // 32, 32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, np.arange(32) ^ o]
    tot = f32(0)
    for s in v[:, 0]:
        tot = f32(tot + s)
    return tot


def _same_bits(got, want):
    assert np.asarray(got, f32).tobytes() == np.asarray(want, f32).tobytes(), (got, want)


class _DevPtr:
    def __init__(self, p, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (p, False),
                                         "version": 3}


def _read(p, n):
    return torch.as_tensor(_DevPtr(p, n), device="cuda").cpu().numpy().copy()


def _capture(monkeypatch, name, arg_index, fields):
    """Wraps the C entry point `name` so that every call records, right after it returns, the
    float arrays {field: length} behind its argument struct (the next kernel may reuse them)."""
    lib = _lib.lib()
    orig = getattr(lib, name)
    seen = []

    def wrapped(*argv):
        rc = orig(*argv)
        a = argv[arg_index]
        a = a if hasattr(a, "_fields_") else a.contents
        seen.append({"batch": a.batch,
                     **{k: _read(getattr(a, k), n(a.batch)) for k, n in fields.items()
                        if getattr(a, k)}})
        return rc

    monkeypatch.setattr(lib, name, wrapped)
    return seen


def _onehot(B, A, gen):
    return torch.nn.functional.one_hot(torch.randint(A, (B,), generator=gen), A).float().cuda()


def _rand(*shape, gen):
    return torch.randn(*shape, generator=gen).cuda()


# ---------------------------------------------------------------- serial tails
@pytest.mark.parametrize("path", ["wgmma", "rows"])
def test_dqn_td_serial_tail(path, monkeypatch):
    """K2 on both paths; B = 1000 leaves a ragged last tile (16 rows, 32 rows on wgmma)."""
    _select_k2(monkeypatch, path)
    B, S, A = 1000, 16, 8
    meta = dict(S=S, A=A, B=B, sizes=[64, 32], acts=["relu", "relu"], gamma=0.99, tau=0.005,
                loss="huber", maxq=True, multi_steps=None, time_diff=False, boost=None,
                double_q=True, lr=1e-3)
    torch.manual_seed(0)
    t = _build_trainer(meta)
    gen = torch.Generator().manual_seed(1)
    act = _onehot(B, A, gen)
    b = dict(state=_rand(B, S, gen=gen), next_state=_rand(B, S, gen=gen),
             reward=_rand(B, 1, gen=gen), time_diff=torch.ones(B, 1, device="cuda"), step=None,
             not_terminal=torch.ones(B, 1, device="cuda"), action=act, next_action=act,
             possible_actions_mask=torch.ones(B, A, device="cuda"),
             possible_next_actions_mask=torch.ones(B, A, device="cuda"))
    rows = 32 if path == "wgmma" else 16
    fields = {"loss_partials": lambda B: -(-B // rows), "loss": lambda B: 1}
    seen_tc = _capture(monkeypatch, "rb200_dqn_td_step_tc", 2, fields)
    seen_rows = _capture(monkeypatch, "rb200_dqn_td_step", 2, fields)
    t.train_batch(_rlt_batch(b, meta), 0)
    _assert_k2(t, path)
    (got,) = seen_tc if path == "wgmma" else seen_rows
    (tot,) = _serial(got["loss_partials"], -(-B // rows))
    _same_bits(got["loss"][0], tot / f32(B))


def test_pdqn_head_serial_tail():
    B = 1000  # 4 blocks of 256 rows, the last one ragged
    gen = torch.Generator().manual_seed(2)
    t = dict(nq=_rand(B, gen=gen), r=_rand(B, gen=gen), q=_rand(B, gen=gen) * 3,
             nt=torch.ones(B, device="cuda"), dz=torch.empty(B, device="cuda"))
    ws = _ws(-(-B // 256))
    a = _lib.PdqnArgsT()
    a.batch, a.max_num_action, a.gamma, a.loss_kind = B, 0, 0.9, _lib.LOSS_HUBER
    a.next_q_target, a.reward, a.not_terminal = t["nq"].data_ptr(), t["r"].data_ptr(), t["nt"].data_ptr()
    a.q_values, a.dz = t["q"].data_ptr(), t["dz"].data_ptr()
    _set_ws(a, ws)
    _call("rb200_pdqn_head", a)
    p = ws["partials"].cpu().numpy()
    (tot,) = _serial(p, len(p))
    _same_bits(ws["loss"].cpu().numpy()[0], tot / f32(B))


def test_cpe_heads_serial_tail():
    B, A, M = 1000, 4, 3
    gen = torch.Generator().manual_seed(3)
    t = dict(ns=_rand(B, A, gen=gen), act=_onehot(B, A, gen), mr=_rand(B, M, gen=gen),
             nt=torch.ones(B, device="cuda"), re=_rand(B, M * A, gen=gen),
             qc=_rand(B, M * A, gen=gen), qct=_rand(B, M * A, gen=gen),
             dzr=torch.empty(B, M * A, device="cuda"), dzq=torch.empty(B, M * A, device="cuda"))
    nblk = -(-B // 256)
    ws = _ws(2 * nblk, 2)
    a = _lib.CpeArgsT()
    a.batch, a.num_actions, a.num_metrics, a.temperature, a.gamma = B, A, M, 1.0, 0.9
    a.loss_kind = _lib.LOSS_HUBER
    a.next_scores, a.action, a.metrics_reward = t["ns"].data_ptr(), t["act"].data_ptr(), t["mr"].data_ptr()
    a.not_terminal, a.reward_est, a.qcpe = t["nt"].data_ptr(), t["re"].data_ptr(), t["qc"].data_ptr()
    a.qcpe_target_next, a.dz_reward, a.dz_qcpe = t["qct"].data_ptr(), t["dzr"].data_ptr(), t["dzq"].data_ptr()
    _set_ws(a, ws)
    _call("rb200_cpe_heads", a)
    tr, tq = _serial(ws["partials"].cpu().numpy(), nblk, ch=2)
    inv = f32(1) / (f32(B) * f32(M))
    _same_bits(ws["loss"].cpu().numpy(), [tr * inv, tq * inv])


@pytest.mark.parametrize("weighted", [False, True])
def test_sac_critic_and_actor_serial_tails(weighted, monkeypatch):
    """SAC with a learned temperature: both critic losses, the actor loss and the alpha gradient
    (the actor kernel's second channel).  B = 1000 leaves a ragged last 16-row tile."""
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import SACTrainer

    B, S, A = 1000, 12, 3
    torch.manual_seed(4)
    opt = lambda: Optimizer__Union.default(lr=1e-3)  # noqa: E731
    t = SACTrainer(GaussianFullyConnectedActor(S, A, [32, 32], ["relu", "relu"]),
                   FullyConnectedCritic(S, A, [32, 32], ["relu", "relu"]),
                   FullyConnectedCritic(S, A, [32, 32], ["relu", "relu"]),
                   rl=RLParameters(gamma=0.99, target_update_rate=0.005),
                   q_network_optimizer=opt(), actor_network_optimizer=opt(),
                   alpha_optimizer=opt(), minibatch_size=B, entropy_temperature=0.1,
                   target_entropy=-float(A)).cuda()
    gen = torch.Generator().manual_seed(5)
    b = dict(state=_rand(B, S, gen=gen), next_state=_rand(B, S, gen=gen),
             action=(torch.rand(B, A, generator=gen) * 1.98 - 0.99).cuda(),
             next_action=torch.zeros(B, A, device="cuda"), reward=_rand(B, 1, gen=gen),
             not_terminal=torch.ones(B, 1, device="cuda"))
    n = -(-B // 16)
    fields = {"loss_partials": lambda B: 2 * n, "loss": lambda B: 2, "alpha_grad": lambda B: 1}
    critic = _capture(monkeypatch, "rb200_ac_critic_step", 5, fields)
    actor = _capture(monkeypatch, "rb200_ac_actor_step", 3, fields)
    w = (0.05 + 0.95 * torch.rand(B, generator=gen)).cuda() if weighted else None
    t.train_batch(_pbatch(b), 0, importance_weights=w)
    (c,), (ac,) = critic, actor
    t1, t2 = _serial(c["loss_partials"], n, ch=2)
    _same_bits(c["loss"], [t1 / f32(B), t2 / f32(B)])
    s, ent = _serial(ac["loss_partials"], n, ch=2)
    invB = f32(1) / f32(B)
    _same_bits(ac["loss"][0], s * invB)
    _same_bits(ac["alpha_grad"][0], -(ent * invB))


# ---------------------------------------------------------------- block tails
@pytest.mark.parametrize("weighted", [False, True])
def test_c51_head_block_tail(weighted):
    """One CTA per row; B = 600 makes the last block's strided loop wrap past 256 twice."""
    B, A, N = 600, 4, 51
    gen = torch.Generator().manual_seed(6)
    t = dict(lnt=_rand(B, A * N, gen=gen), lc=_rand(B, A * N, gen=gen), act=_onehot(B, A, gen),
             r=_rand(B, gen=gen), nt=torch.ones(B, device="cuda"),
             sup=torch.linspace(-10, 10, N, device="cuda"), dz=torch.empty(B, A * N, device="cuda"),
             w=(0.05 + 0.95 * torch.rand(B, generator=gen)).cuda())
    ws = _ws(B)
    a = _lib.C51ArgsT()
    a.batch, a.num_actions, a.num_atoms, a.gamma, a.maxq, a.double_q = B, A, N, 0.9, 1, 0
    a.qmin, a.qmax, a.scale_support = -10.0, 10.0, 20.0 / (N - 1)
    a.logits_next_target, a.logits_cur, a.action = t["lnt"].data_ptr(), t["lc"].data_ptr(), t["act"].data_ptr()
    a.reward, a.not_terminal, a.support = t["r"].data_ptr(), t["nt"].data_ptr(), t["sup"].data_ptr()
    a.dz_logits = t["dz"].data_ptr()
    a.sample_weight = t["w"].data_ptr() if weighted else None
    _set_ws(a, ws)
    _call("rb200_c51_head", a)
    w = t["w"].cpu().numpy() if weighted else None
    tot = _block(ws["partials"].cpu().numpy(), B, w)
    _same_bits(ws["loss"].cpu().numpy()[0], tot * (f32(1) / f32(B)))


@pytest.mark.parametrize("weighted", [False, True])
def test_qr_head_block_tail(weighted):
    B, A, N = 600, 4, 32
    gen = torch.Generator().manual_seed(7)
    t = dict(qnt=_rand(B, A * N, gen=gen), qc=_rand(B, A * N, gen=gen), act=_onehot(B, A, gen),
             r=_rand(B, gen=gen), nt=torch.ones(B, device="cuda"),
             dz=torch.empty(B, A * N, device="cuda"),
             w=(0.05 + 0.95 * torch.rand(B, generator=gen)).cuda())
    ws = _ws(B)
    a = _lib.QrdqnArgsT()
    a.batch, a.num_actions, a.num_atoms, a.gamma, a.maxq, a.double_q = B, A, N, 0.9, 1, 0
    a.q_next_target, a.q_cur, a.action = t["qnt"].data_ptr(), t["qc"].data_ptr(), t["act"].data_ptr()
    a.reward, a.not_terminal, a.dz_head = t["r"].data_ptr(), t["nt"].data_ptr(), t["dz"].data_ptr()
    a.sample_weight = t["w"].data_ptr() if weighted else None
    _set_ws(a, ws)
    _call("rb200_qrdqn_head", a)
    w = t["w"].cpu().numpy() if weighted else None
    tot = _block(ws["partials"].cpu().numpy(), B, w)
    norm = f32(1) / (f32(N) * f32(B) * f32(N))
    _same_bits(ws["loss"].cpu().numpy()[0], tot * norm)


def test_bc_xent_head_block_tail():
    """8 rows per block: B = 2501 gives 313 blocks, the last one with a single row."""
    B, A = 2501, 6
    gen = torch.Generator().manual_seed(8)
    t = dict(x=_rand(B, A, gen=gen), lab=_onehot(B, A, gen), m=torch.ones(B, A, device="cuda"),
             dz=torch.empty(B, A, device="cuda"))
    nblk = -(-B // _lib.BC_ROWS_PER_BLOCK)
    ws = _ws(nblk)
    a = _lib.BcXentArgsT()
    a.batch, a.num_actions = B, A
    a.logits, a.labels, a.mask, a.dz = (t["x"].data_ptr(), t["lab"].data_ptr(), t["m"].data_ptr(),
                                        t["dz"].data_ptr())
    _set_ws(a, ws)
    _call("rb200_bc_xent_head", a)
    tot = _block(ws["partials"].cpu().numpy(), nblk)
    _same_bits(ws["loss"].cpu().numpy()[0], tot / f32(B))
