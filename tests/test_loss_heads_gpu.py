"""The row-local loss heads and the dueling fold called through the C ABI and compared with the
float64 restatements of oracle/heads_fp64.py (pinned to td_oracle by test_loss_heads_cpu.py)
at the shapes and values where they go wrong:

* qr_head_kernel: actions beyond the 64 staged ones, N % 4 != 0 and misaligned inputs (scalar
  loads), N > 256 (several atoms per thread), N at the 48 KB limit, SARSA, masks, TD errors of
  exactly 0 and +-1, importance weights, NaN targets, a missing q_next_online.
* c51_head_kernel: A * N past the 48 KB opt-in and at the 200 KB cap, exact-grid projections
  that reach every l == u rule, exact arg-max ties, supports where (qmax - qmin) / scale lands
  an ulp above N - 1, NaN targets.
* pdqn_head_kernel and cpe_heads_kernel: ragged batches, masks, both losses at |delta| = 1,
  the POW discount, temperature != 1, fully masked rows, ties in the logged action.
* rb200_dueling_fold / rb200_dueling_unfold: R = A * N > 1024, H not a multiple of 32, several
  gradient slabs at offsets that leave gaps.
* C51Trainer and QRDQNTrainer on a dueling network with atoms over two updates.

Every output is compared per tensor at 1e-5 relative; NaN must sit exactly where the reference
has it.  next_action_idx must equal the fp64 arg max except on rows whose two best values lie
within 1e-5 relative, where the kernel's choice is fed to the reference.  Each launch runs twice
and must give bit-identical outputs."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import heads_fp64 as H
from reagent_b200 import _lib
from tests import golden_util as G
from tests.kernel_util import _call, _set_ws, _ws

pytestmark = pytest.mark.gpu

TOL = 1e-5
NAN = float("nan")
E_INVALID, E_SMEM = -1, -3
f32 = np.float32


def _close(got, want, what, tol=TOL):
    got = torch.as_tensor(got, dtype=torch.float64).cpu().reshape(-1)
    want = torch.as_tensor(want, dtype=torch.float64).cpu().reshape(-1)
    assert torch.equal(got.isnan(), want.isnan()), (what, "NaN positions differ")
    fin = ~want.isnan()
    if fin.any():
        err = G.rel_err(got[fin], want[fin])
        assert err < tol, (what, err)


def _cuda(t, offset=0):
    """`t` as a contiguous fp32 (or int) CUDA tensor starting `offset` elements into its
    allocation (offset 1 breaks the 16-byte alignment)."""
    if t is None:
        return None
    t = t.contiguous()
    buf = torch.full((t.numel() + offset,), NAN if t.is_floating_point() else 0, dtype=t.dtype,
                     device="cuda")
    buf[offset:] = t.reshape(-1).cuda()
    return buf[offset:].view(t.shape)


def _launch(fn, Args, ins, outs, n_partials, n_loss=1, **scalars):
    """Runs entry point `fn` twice on the same inputs and requires bit-identical outputs.
    ins: {field: CUDA tensor | None}; outs: {field: (shape, dtype) | None}; returns the outputs,
    loss_partials and loss on the CPU."""
    res = []
    for _ in range(2):
        a = Args()
        for k, v in scalars.items():
            setattr(a, k, v)
        for k, v in ins.items():
            setattr(a, k, None if v is None else v.data_ptr())
        bufs = {}
        for k, spec in outs.items():
            if spec is None:
                setattr(a, k, None)
                continue
            shape, dt = spec
            bufs[k] = torch.full(shape, NAN if dt.is_floating_point else -7, dtype=dt, device="cuda")
            setattr(a, k, bufs[k].data_ptr())
        ws = _ws(n_partials, n_loss)
        _set_ws(a, ws)
        _call(fn, a)
        r = {k: v.cpu() for k, v in bufs.items()}
        r["loss_partials"], r["loss"] = ws["partials"].cpu(), ws["loss"].cpu()
        res.append(r)
    for k in res[0]:
        assert res[0][k].numpy().tobytes() == res[1][k].numpy().tobytes(), (fn, k, "not deterministic")
    return res[0]


def _rc(fn, Args, **fields):
    """Return code of one call whose arguments are rejected before any launch."""
    a = Args()
    for k, v in fields.items():
        setattr(a, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    ws = _ws(1)
    _set_ws(a, ws)
    return getattr(_lib.lib(), fn)(C.byref(a), _lib.cur_stream())


def _with_kernel_choice(ref_fn, kernel_idx):
    """fp64 reference with the arg max checked against the kernel's: equal off the near-tie
    rows, a near-maximal action on them (then the kernel's choice is fed to the reference).
    Returns (reference outputs, number of near-tie rows)."""
    ref = ref_fn(None)
    if ref["next_action_idx"] is None:
        return ref, 0
    qv = ref["next_q_values"]
    k = kernel_idx.to(torch.int64).reshape(-1)
    tie = H.argmax_near_ties(qv)
    assert torch.equal(k[~tie], ref["next_action_idx"][~tie]), "arg max differs off the near ties"
    assert bool(((k >= 0) & (k < qv.shape[1])).all())
    top = qv.max(1).values
    near = (top - qv.gather(1, k.clamp(0, qv.shape[1] - 1)[:, None])[:, 0]) <= 1e-5 * top.abs()
    assert bool(near[tie].all()), "the kernel's choice on a near tie is not near maximal"
    if tie.any():
        ref = ref_fn(k)
    return ref, int(tie.sum())


def _onehot(B, A, gen):
    return torch.nn.functional.one_hot(torch.randint(A, (B,), generator=gen), A).float()


def _mask(kind, B, A, gen, sel_means=None, full_row=True):
    """None (all allowed) | "partial" (random, the best action of the selection net masked out
    on every other row, row 0 fully masked if full_row) | "zero" (every row fully masked)."""
    if kind is None:
        return None
    if kind == "zero":
        return torch.zeros(B, A)
    m = (torch.rand(B, A, generator=gen) < 0.6).float()
    if sel_means is not None and A > 1:
        best = sel_means.argmax(1)
        m[torch.arange(0, B, 2), best[0::2]] = 0.0
    m[torch.arange(B), torch.randint(A, (B,), generator=gen)] = 1.0
    if full_row:
        m[0] = 0.0
    return m


# ---------------------------------------------------------------------------------- QR-DQN
QR_CASES = [
    # id, B, A, N, options
    ("b1_a1_n1", 1, 1, 1, dict()),
    ("a64_n31_masked", 257, 64, 31, dict(mask="partial", exact_td=True, terminal=True)),
    ("a65_n3_unstaged", 257, 65, 3, dict(mask="partial", boost=True, disc=True)),
    ("a200_n2_unstaged_single", 257, 200, 2, dict(double_q=False, mask="partial")),
    ("a4_n257_weighted", 257, 4, 257, dict(weighted=True, exact_td=True)),
    ("n_at_48k", 1, 3, 6014, dict(disc=True)),
    ("b4096_a32_n200_weighted", 4096, 32, 200, dict(weighted=True, mask="partial", terminal=True)),
    ("n64_aligned", 257, 8, 64, dict(boost=True)),
    ("n64_misaligned", 257, 8, 64, dict(boost=True, offset=1)),
    ("sarsa_single", 257, 5, 16, dict(maxq=False, double_q=False, terminal=True, exact_td=True)),
    ("sarsa_double", 257, 66, 5, dict(maxq=False, disc=True, boost=True)),
    ("all_masked", 33, 6, 8, dict(mask="zero")),
]


def _qr_inputs(B, A, N, seed, o):
    gen = torch.Generator().manual_seed(seed)
    t = dict(q_next_online=torch.randn(B, A * N, generator=gen),
             q_next_target=torch.randn(B, A * N, generator=gen),
             q_cur=torch.randn(B, A * N, generator=gen), action=_onehot(B, A, gen),
             next_action=_onehot(B, A, gen), reward=torch.randn(B, generator=gen),
             not_terminal=(torch.rand(B, generator=gen) > 0.25).float() if o.get("terminal")
             else torch.ones(B),
             discount_src=torch.randint(1, 4, (B,), generator=gen).float() if o.get("disc") else None,
             reward_boost=torch.randn(A, generator=gen) if o.get("boost") else None,
             sample_weight=(0.05 + 0.95 * torch.rand(B, generator=gen)) if o.get("weighted") else None)
    sel = t["q_next_online"] if o.get("double_q", True) else t["q_next_target"]
    t["possible_next_actions_mask"] = _mask(o.get("mask"), B, A, gen, sel.view(B, A, N).mean(2))
    if o.get("exact_td"):  # terminal rows with target 0.5: TD errors of exactly 0, +1 and -1
        for b in range(min(B, 4)):
            t["not_terminal"][b], t["reward"][b] = 0.0, 0.5
            a = int(t["action"][b].argmax())
            t["q_cur"][b, a * N:(a + 1) * N] = torch.tensor([0.5, -0.5, 1.5]).repeat(N)[:N]
    return t


def _qr_run(t, B, A, N, *, double_q, maxq, offset=0):
    ins = {k: _cuda(v, offset if k in ("q_next_online", "q_next_target", "q_cur") else 0)
           for k, v in t.items()}
    if not maxq:
        ins["possible_next_actions_mask"] = None
    outs = dict(dz_head=((B, A * N), torch.float32), all_q_values=((B, A), torch.float32),
                next_action_idx=((B,), torch.int32))
    return _launch("rb200_qrdqn_head", _lib.QrdqnArgsT, ins, outs, B, batch=B, num_actions=A,
                   num_atoms=N, gamma=0.9, double_q=int(double_q), maxq=int(maxq))


def _qr_ref(t, N, *, double_q, maxq, next_idx=None):
    return H.qr_head(t["q_next_online"], t["q_next_target"], t["q_cur"], t["action"],
                     t["next_action"], t["possible_next_actions_mask"] if maxq else None,
                     t["reward"], t["not_terminal"], num_atoms=N, gamma=f32(0.9),
                     double_q=double_q, maxq=maxq, discount_src=t["discount_src"],
                     reward_boost=t["reward_boost"], sample_weight=t["sample_weight"],
                     next_idx=next_idx, row_chunk=max(1, 2 ** 23 // (N * N)))


def _qr_compare(got, ref, maxq, N):
    # each dz_head entry and row loss is a float32 sum over two chains of N / 2 pairs: 1e-5
    # holds to N = 512, beyond that the accumulators' rounding grows with the chain length
    # (measured on an H100 at N = 6014: 3.5e-5 for dz_head)
    tol = TOL * max(1.0, N / 512)
    _close(got["dz_head"], ref["dz"], "dz_head", tol)
    _close(got["loss_partials"], ref["loss_partials"], "loss_partials", tol)
    _close(got["loss"], ref["loss"], "loss", tol)
    _close(got["all_q_values"], ref["all_q_values"], "all_q_values")
    if not maxq:
        assert bool((got["next_action_idx"] == 0).all())  # SARSA: the kernel writes 0


@pytest.mark.parametrize("case", QR_CASES, ids=[c[0] for c in QR_CASES])
def test_qr_head_kernel_matches_fp64(case):
    name, B, A, N, o = case
    double_q, maxq = o.get("double_q", True), o.get("maxq", True)
    t = _qr_inputs(B, A, N, sum(map(ord, name)), o)
    got = _qr_run(t, B, A, N, double_q=double_q, maxq=maxq, offset=o.get("offset", 0))
    ref, ties = _with_kernel_choice(
        lambda idx: _qr_ref(t, N, double_q=double_q, maxq=maxq, next_idx=idx), got["next_action_idx"])
    if o.get("mask") != "zero":
        assert ties <= max(1, B // 50), ties
    _qr_compare(got, ref, maxq, N)


def test_qr_head_nan_target_gives_nan_gradient():
    """A NaN reward or not_terminal: that row's loss, loss_partials entry and whole dz_head row
    are NaN (autograd's Huber derivative keeps the NaN); every other row is bit-identical to a
    run without the NaN."""
    B, A, N = 40, 5, 12
    t = _qr_inputs(B, A, N, 11, dict(terminal=True))
    clean = _qr_run(t, B, A, N, double_q=True, maxq=True)
    t["reward"][3], t["not_terminal"][17] = NAN, NAN
    got = _qr_run(t, B, A, N, double_q=True, maxq=True)
    ref, _ = _with_kernel_choice(lambda idx: _qr_ref(t, N, double_q=True, maxq=True, next_idx=idx),
                                 got["next_action_idx"])
    _qr_compare(got, ref, True, N)
    bad = torch.zeros(B, dtype=torch.bool)
    bad[[3, 17]] = True
    assert bool(got["dz_head"][bad].isnan().all()) and bool(got["loss_partials"][bad].isnan().all())
    assert bool(got["loss"].isnan().all())
    for k in ("dz_head", "loss_partials", "all_q_values", "next_action_idx"):
        assert got[k][~bad].numpy().tobytes() == clean[k][~bad].numpy().tobytes(), k


def test_qr_head_double_q_requires_online_logits():
    """double_q reads the atom means of q_next_online even for SARSA: without the pointer the
    call is rejected, for SARSA as for max-Q."""
    B, A, N = 4, 3, 5
    t = {k: _cuda(v) for k, v in _qr_inputs(B, A, N, 0, {}).items()}
    dz = torch.empty(B, A * N, device="cuda")
    for maxq in (0, 1):
        rc = _rc("rb200_qrdqn_head", _lib.QrdqnArgsT, batch=B, num_actions=A, num_atoms=N,
                 q_next_target=t["q_next_target"], q_cur=t["q_cur"], action=t["action"],
                 next_action=t["next_action"], reward=t["reward"], not_terminal=t["not_terminal"],
                 gamma=0.9, double_q=1, maxq=maxq, dz_head=dz)
        assert rc == E_INVALID, (maxq, rc)


def test_qr_head_rejects_atoms_past_48k():
    B, A, N = 1, 1, 6016  # (2 N + A + 256) floats = 48 KB + 4 bytes
    t = {k: _cuda(v) for k, v in _qr_inputs(B, A, N, 0, {}).items()}
    rc = _rc("rb200_qrdqn_head", _lib.QrdqnArgsT, batch=B, num_actions=A, num_atoms=N,
             q_next_online=t["q_next_online"], q_next_target=t["q_next_target"], q_cur=t["q_cur"],
             action=t["action"], reward=t["reward"], not_terminal=t["not_terminal"], gamma=0.9,
             double_q=1, maxq=1, dz_head=torch.empty(B, A * N, device="cuda"))
    assert rc == E_SMEM


# ---------------------------------------------------------------------------------- C51
C51_CASES = [
    ("a1_n2_sarsa", 3, 1, 2, dict(maxq=False, double_q=False)),
    ("a2_n51_masked", 64, 2, 51, dict(mask="partial", terminal=True)),
    ("a32_n101_weighted", 50, 32, 101, dict(weighted=True, boost=True, disc=True)),
    ("a33_n51_single", 33, 33, 51, dict(double_q=False, mask="partial")),
    ("a33_n2_sarsa_double", 40, 33, 2, dict(maxq=False, boost=True, terminal=True)),
    ("a64_n101_past_48k", 20, 64, 101, dict(mask="partial", weighted=True)),
    ("a167_n101_at_200k", 4, 167, 101, dict(terminal=True)),
    ("all_masked", 9, 4, 51, dict(mask="zero")),
]


def _c51_inputs(B, A, N, seed, o, qmin=-10.0, qmax=10.0):
    gen = torch.Generator().manual_seed(seed)
    t = dict(logits_next_online=torch.randn(B, A * N, generator=gen) * 2,
             logits_next_target=torch.randn(B, A * N, generator=gen) * 2,
             logits_cur=torch.randn(B, A * N, generator=gen) * 2, action=_onehot(B, A, gen),
             next_action=_onehot(B, A, gen), reward=torch.randn(B, generator=gen) * 4,
             not_terminal=(torch.rand(B, generator=gen) > 0.25).float() if o.get("terminal")
             else torch.ones(B),
             discount_src=torch.randint(1, 4, (B,), generator=gen).float() if o.get("disc") else None,
             reward_boost=torch.randn(A, generator=gen) if o.get("boost") else None,
             sample_weight=(0.05 + 0.95 * torch.rand(B, generator=gen)) if o.get("weighted") else None,
             support=torch.linspace(qmin, qmax, N))
    sel = torch.softmax((t["logits_next_online"] if o.get("double_q", True)
                         else t["logits_next_target"]).view(B, A, N), -1) @ t["support"]
    t["possible_next_actions_mask"] = _mask(o.get("mask"), B, A, gen, sel)
    return t


def _c51_run(t, B, A, N, *, double_q, maxq, qmin=-10.0, qmax=10.0):
    ins = {k: _cuda(v) for k, v in t.items()}
    if not maxq:
        ins["possible_next_actions_mask"] = None
    outs = dict(dz_logits=((B, A * N), torch.float32), all_q_values=((B, A), torch.float32),
                next_action_idx=((B,), torch.int32) if maxq else None)
    return _launch("rb200_c51_head", _lib.C51ArgsT, ins, outs, B, batch=B, num_actions=A,
                   num_atoms=N, gamma=0.9, qmin=qmin, qmax=qmax,
                   scale_support=(qmax - qmin) / (N - 1.0), double_q=int(double_q), maxq=int(maxq))


def _c51_ref(t, *, double_q, maxq, qmin=-10.0, qmax=10.0, next_idx=None):
    N = t["support"].numel()
    return H.c51_head(t["logits_next_online"], t["logits_next_target"], t["logits_cur"],
                      t["action"], t["next_action"], t["possible_next_actions_mask"] if maxq else None,
                      t["reward"], t["not_terminal"], t["support"], gamma=f32(0.9), qmin=qmin,
                      qmax=qmax, scale_support=f32((qmax - qmin) / (N - 1.0)), double_q=double_q,
                      maxq=maxq, discount_src=t["discount_src"], reward_boost=t["reward_boost"],
                      sample_weight=t["sample_weight"], next_idx=next_idx)


def _c51_check(t, B, A, N, *, double_q=True, maxq=True, qmin=-10.0, qmax=10.0, max_ties=None,
               all_q=True):
    got = _c51_run(t, B, A, N, double_q=double_q, maxq=maxq, qmin=qmin, qmax=qmax)
    idx = got["next_action_idx"] if maxq else torch.zeros(B, dtype=torch.int32)
    ref, ties = _with_kernel_choice(
        lambda i: _c51_ref(t, double_q=double_q, maxq=maxq, qmin=qmin, qmax=qmax, next_idx=i), idx)
    if max_ties is not None:
        assert ties <= max_ties, ties
    _close(got["dz_logits"], ref["dz"], "dz_logits")
    _close(got["loss_partials"], ref["loss_partials"], "loss_partials")
    _close(got["loss"], ref["loss"], "loss")
    if all_q:
        _close(got["all_q_values"], ref["all_q_values"], "all_q_values")
    return got, ref


@pytest.mark.parametrize("case", C51_CASES, ids=[c[0] for c in C51_CASES])
def test_c51_head_kernel_matches_fp64(case):
    name, B, A, N, o = case
    t = _c51_inputs(B, A, N, sum(map(ord, name)), o)
    _c51_check(t, B, A, N, double_q=o.get("double_q", True), maxq=o.get("maxq", True),
               max_ties=None if o.get("mask") == "zero" else max(1, B // 50))


def test_c51_head_rejects_past_200k():
    B, A, N = 1, 168, 101  # 3 A N + 2 N + A floats > 200 KB
    t = {k: _cuda(v) for k, v in _c51_inputs(B, A, N, 0, {}).items()}
    rc = _rc("rb200_c51_head", _lib.C51ArgsT, batch=B, num_actions=A, num_atoms=N,
             logits_next_online=t["logits_next_online"], logits_next_target=t["logits_next_target"],
             logits_cur=t["logits_cur"], action=t["action"], reward=t["reward"],
             not_terminal=t["not_terminal"], support=t["support"], gamma=0.9, qmin=-10.0,
             qmax=10.0, scale_support=0.2, double_q=1, maxq=1,
             dz_logits=torch.empty(B, A * N, device="cuda"))
    assert rc == E_SMEM


@pytest.mark.parametrize("maxq", [True, False])
def test_c51_head_exact_grid_projection(maxq):
    """qmin -10, qmax 10, N 41: scale 0.5, so b is an exact integer or half-integer in fp32 and
    fp64 alike.  Terminal rows whose reward sits on atom 0, on interior atoms, on atom N - 1 and
    beyond both ends reach each l == u rule; gamma 0.5 on non-terminal rows lands the targets
    on quarter steps of the grid."""
    B, A, N = 16, 3, 41
    t = _c51_inputs(B, A, N, 5, {})
    rewards = [-10.0, -9.5, 0.0, 3.0, 9.5, 10.0, -15.0, 15.0, -10.0, 0.0, 10.0, 2.5, -0.5, 7.0, 20.0, -20.0]
    t["reward"] = torch.tensor(rewards)
    t["not_terminal"] = torch.tensor([0.0] * 8 + [1.0] * 8)
    t["discount_src"] = None
    gamma = 0.5
    got = _launch("rb200_c51_head", _lib.C51ArgsT, {k: _cuda(v) for k, v in t.items()},
                  dict(dz_logits=((B, A * N), torch.float32), all_q_values=((B, A), torch.float32),
                       next_action_idx=((B,), torch.int32) if maxq else None),
                  B, batch=B, num_actions=A, num_atoms=N, gamma=gamma, qmin=-10.0, qmax=10.0,
                  scale_support=0.5, double_q=1, maxq=int(maxq))
    idx = got["next_action_idx"] if maxq else torch.zeros(B, dtype=torch.int32)
    ref, _ = _with_kernel_choice(
        lambda i: H.c51_head(t["logits_next_online"], t["logits_next_target"], t["logits_cur"],
                             t["action"], t["next_action"], None, t["reward"], t["not_terminal"],
                             t["support"], gamma=gamma, qmin=-10.0, qmax=10.0, scale_support=0.5,
                             double_q=True, maxq=maxq, next_idx=i), idx)
    b = (ref["m"] != 0).nonzero()
    assert {0, N - 1} <= set(b[:, 1].tolist())  # mass reaches both end atoms
    _close(got["dz_logits"], ref["dz"], "dz_logits")
    _close(got["loss_partials"], ref["loss_partials"], "loss_partials")
    _close(got["loss"], ref["loss"], "loss")


def test_c51_head_exact_tie_takes_first_action():
    """Duplicate action rows in the selection network: equal expected values in fp32, and the
    first index wins as in torch.argmax."""
    B, A, N = 24, 5, 51
    t = _c51_inputs(B, A, N, 9, {})
    for key in ("logits_next_online", "logits_next_target"):
        x = t[key].view(B, A, N)
        x[:, 3] = x[:, 1]
        x[:, 4] = x[:, 1]
    lo = t["logits_next_online"].view(B, A, N)
    lo[:, 1] += 1.0  # make the duplicated action the best one on every row
    lo[:, 3] = lo[:, 1]
    lo[:, 4] = lo[:, 1]
    got, ref = _c51_check(t, B, A, N, double_q=True, maxq=True)
    best = H.c51_head(t["logits_next_online"], t["logits_next_target"], t["logits_cur"], t["action"],
                      None, None, t["reward"], t["not_terminal"], t["support"], gamma=0.9,
                      qmin=-10.0, qmax=10.0, scale_support=0.5, double_q=True, maxq=True)
    tied = best["next_action_idx"] == 1
    assert bool(tied.any())
    assert bool((got["next_action_idx"][tied] == 1).all())


@pytest.mark.parametrize("qmin,qmax,N", [(-10.0, 10.0, 124), (-3.0, 5.0, 62)])
def test_c51_head_support_past_last_atom(qmin, qmax, N):
    """In fp32 (qmax - qmin) / scale_support is an ulp above N - 1 on these supports: the
    projection of a target at qmax must stay on atom N - 1 and keep all of next_dist's mass.
    With uniform current logits the row cross entropy is log(N) * sum(m)."""
    B, A = 12, 3
    t = _c51_inputs(B, A, N, 13, {}, qmin=qmin, qmax=qmax)
    assert f32(f32(qmax) - f32(qmin)) / f32((qmax - qmin) / (N - 1.0)) > N - 1
    t["logits_cur"] = torch.zeros(B, A * N)
    t["reward"][: B // 2] = qmax + 1.0  # all of the row's targets at qmax (terminal rows)
    t["not_terminal"][: B // 2] = 0.0
    t["reward"][B // 2:] = qmax  # and on non-terminal rows, the upper part of the support
    # (all_q_values: the support's mean, about 0 -- covered by the other C51 tests)
    got, ref = _c51_check(t, B, A, N, qmin=qmin, qmax=qmax, all_q=False)
    msum = got["loss_partials"].double() / np.log(N)
    assert float((msum - 1.0).abs().max()) < 1e-6, msum
    assert float((ref["m"].sum(1) - ref["next_dist"].sum(1)).abs().max()) < 1e-12


def test_c51_head_nan_target_propagates():
    """A NaN reward, not_terminal or discount: that row's projection, loss_partials entry and
    dz_logits are NaN and so is the loss; every other row is bit-identical to a run without
    the NaNs."""
    B, A, N = 30, 4, 51
    t = _c51_inputs(B, A, N, 17, dict(disc=True, terminal=True))
    clean = _c51_run(t, B, A, N, double_q=True, maxq=True)
    t["reward"][2], t["not_terminal"][9], t["discount_src"][20] = NAN, NAN, NAN
    got, _ = _c51_check(t, B, A, N)
    bad = torch.zeros(B, dtype=torch.bool)
    bad[[2, 9, 20]] = True
    assert bool(got["loss_partials"][bad].isnan().all()) and bool(got["loss"].isnan().all())
    taken = t["action"].repeat_interleave(N, 1).bool()
    assert bool(got["dz_logits"][bad][taken[bad]].isnan().all())
    for k in ("dz_logits", "loss_partials", "all_q_values", "next_action_idx"):
        assert got[k][~bad].numpy().tobytes() == clean[k][~bad].numpy().tobytes(), k


# ---------------------------------------------------------------------------------- ParametricDQN
PDQN_CASES = [(M, B, mask, dq, loss)
              for M, B, mask, dq, loss in [
                  (0, 1, None, False, "mse"), (0, 257, None, False, "huber"),
                  (1, 255, None, True, "mse"), (1, 257, "partial", True, "huber"),
                  (7, 1000, "partial", True, "mse"), (7, 257, "zero", True, "huber"),
                  (7, 255, "partial", "no_next_q", "huber"), (64, 1000, "partial", False, "mse"),
                  (64, 257, None, True, "huber"), (64, 1, "partial", True, "mse")]]


@pytest.mark.parametrize("pow_discount", [False, True])
@pytest.mark.parametrize("M,B,mask,double_q,loss", PDQN_CASES)
def test_pdqn_head_kernel_matches_fp64(M, B, mask, double_q, loss, pow_discount):
    gen = torch.Generator().manual_seed(M * 7919 + B)
    n = max(M, 1) * B
    t = dict(next_q=torch.randn(n, generator=gen) if M and double_q is True else None,
             next_q_target=torch.randn(n, generator=gen),
             mask=_mask(mask, B, M, gen, full_row=False) if M else None,
             reward=torch.randn(B, generator=gen), not_terminal=(torch.rand(B, generator=gen) > 0.2).float(),
             discount_src=torch.randint(1, 5, (B,), generator=gen).float() if pow_discount else None,
             q_values=torch.randn(B, generator=gen) * 2)
    # |delta| exactly 1 (and 0) on terminal rows: q = reward + {1, -1, 0}
    for b, d in zip(range(min(B, 3)), (1.0, -1.0, 0.0)):
        t["not_terminal"][b], t["reward"][b] = 0.0, 0.25
        t["q_values"][b] = 0.25 + d
    got = _launch("rb200_pdqn_head", _lib.PdqnArgsT, {k: _cuda(v) for k, v in t.items()},
                  dict(dz=((B,), torch.float32), td_target=((B,), torch.float32)),
                  -(-B // 256), batch=B, max_num_action=M, gamma=0.9,
                  discount_mode=_lib.DISCOUNT_POW if pow_discount else _lib.DISCOUNT_CONST,
                  double_q=int(bool(double_q)),
                  loss_kind=_lib.LOSS_HUBER if loss == "huber" else _lib.LOSS_MSE)
    ref = H.pdqn_head(t["next_q"], t["next_q_target"], t["mask"], t["reward"], t["not_terminal"],
                      t["q_values"], max_num_action=M, gamma=f32(0.9), double_q=bool(double_q),
                      loss=loss, discount_src=t["discount_src"])
    # fully masked rows: the -1e9 penalty reaches the target of the non-terminal rows, so the
    # terminal rows (target = reward) are compared on their own scale
    groups = [t["not_terminal"] == 0, t["not_terminal"] != 0] if mask == "zero" else [slice(None)]
    for g in groups:
        _close(got["td_target"][g], ref["td_target"][g], "td_target")
        _close(got["dz"][g], ref["dz"][g], "dz")
    _close(got["loss"], ref["loss"], "loss")


# ---------------------------------------------------------------------------------- CPE
@pytest.mark.parametrize("loss", ["mse", "huber"])
@pytest.mark.parametrize("mask", [None, "partial", "rows_zero"])
@pytest.mark.parametrize("A,M", [(1, 1), (2, 3), (17, 1), (17, 3)])
def test_cpe_heads_kernel_matches_fp64(A, M, mask, loss):
    B = 300
    gen = torch.Generator().manual_seed(A * 100 + M)
    act = _onehot(B, A, gen)
    act[: B // 10] = 0.0  # logged-action ties: all-zero rows (first index) and duplicated maxima
    if A > 1:
        act[B // 10: B // 5, :2] = 1.0
    msk = None
    if mask is not None:
        msk = (torch.rand(B, A, generator=gen) < 0.6).float()
        msk[torch.arange(B), torch.randint(A, (B,), generator=gen)] = 1.0
        if mask == "rows_zero":
            msk[::7] = 0.0  # fully masked rows: propensity 0
    t = dict(next_scores=torch.randn(B, A, generator=gen) * 3, mask=msk, action=act,
             metrics_reward=torch.randn(B, M, generator=gen),
             discount_src=torch.randint(1, 4, (B,), generator=gen).float(),
             not_terminal=(torch.rand(B, generator=gen) > 0.2).float(),
             reward_est=torch.randn(B, M * A, generator=gen),
             qcpe=torch.randn(B, M * A, generator=gen) * 2,
             qcpe_target_next=torch.randn(B, M * A, generator=gen))
    got = _launch("rb200_cpe_heads", _lib.CpeArgsT, {k: _cuda(v) for k, v in t.items()},
                  dict(dz_reward=((B, M * A), torch.float32), dz_qcpe=((B, M * A), torch.float32),
                       propensities_next=((B, A), torch.float32)),
                  2 * -(-B // 256), 2, batch=B, num_actions=A, num_metrics=M, temperature=0.35,
                  gamma=0.9, discount_mode=_lib.DISCOUNT_POW,
                  loss_kind=_lib.LOSS_HUBER if loss == "huber" else _lib.LOSS_MSE)
    ref = H.cpe_heads(t["next_scores"], t["mask"], t["action"], t["metrics_reward"],
                      t["not_terminal"], t["reward_est"], t["qcpe"], t["qcpe_target_next"],
                      temperature=float(f32(0.35)), gamma=f32(0.9), loss=loss, discount_src=t["discount_src"])
    _close(got["propensities_next"], ref["propensities_next"], "propensities_next")
    _close(got["dz_reward"], ref["dz_reward"], "dz_reward")
    _close(got["dz_qcpe"], ref["dz_qcpe"], "dz_qcpe")
    _close(got["loss"], ref["loss"], "loss")
    if mask == "rows_zero":
        assert bool((got["propensities_next"][::7] == 0).all())
    off = torch.ones(B, M, A, dtype=torch.bool)
    off[torch.arange(B), :, ref["logged"]] = False
    for k in ("dz_reward", "dz_qcpe"):
        assert bool((got[k].view(B, M, A)[off] == 0).all()), k


# ---------------------------------------------------------------------------------- dueling
DUELING_SHAPES = [(1, 1, 1), (2, 1, 31), (4, 1, 33), (3, 51, 100), (65, 7, 256), (32, 200, 128)]


@pytest.mark.parametrize("A,N,Hh", DUELING_SHAPES)
def test_dueling_fold_matches_fp64(A, N, Hh):
    gen = torch.Generator().manual_seed(A * 1000 + N + Hh)
    R = A * N
    p = [torch.randn(R, Hh, generator=gen), torch.randn(R, generator=gen),
         torch.randn(N, Hh, generator=gen), torch.randn(N, generator=gen)]
    d = [_cuda(x) for x in p]
    lib = _lib.lib()
    scratch = torch.empty(lib.rb200_dueling_scratch_floats(Hh, 1), device="cuda")
    outs = []
    for _ in range(2):
        W_q = torch.full((R, 2 * Hh), NAN, device="cuda")
        b_q = torch.full((R,), NAN, device="cuda")
        _lib.check(lib.rb200_dueling_fold(*[x.data_ptr() for x in d], A, N, Hh, W_q.data_ptr(),
                                          b_q.data_ptr(), scratch.data_ptr(), _lib.cur_stream()),
                   "rb200_dueling_fold")
        torch.cuda.synchronize()
        outs.append((W_q.cpu(), b_q.cpu()))
    assert all(torch.equal(x, y) for x, y in zip(outs[0], outs[1]))
    W_ref, b_ref = H.dueling_fold(*[x.double() for x in p], A, N)
    _close(outs[0][0], W_ref, "W_q")
    _close(outs[0][1], b_ref, "b_q")


@pytest.mark.parametrize("splits", [1, 3, 16])
@pytest.mark.parametrize("A,N,Hh", DUELING_SHAPES)
def test_dueling_unfold_matches_fp64(A, N, Hh, splits):
    """Per slab: random folded gradients mapped back by the transposed linear map; the folded
    gradient is zero afterwards and the sentinel-filled gaps between the regions untouched."""
    gen = torch.Generator().manual_seed(A * 1000 + N + Hh + splits)
    R = A * N
    sizes = [("W_q", R * 2 * Hh), ("b_q", R), ("W_adv", R * Hh), ("b_adv", R), ("w_val", N * Hh),
             ("b_val", N)]
    off, o = {}, 3
    for k, n in sizes:
        off[k] = o
        o += n + 5  # a 5-float gap after each region
    stride = o + 7
    SENT = 12345.0
    g = torch.full((splits, stride), SENT)
    for s in range(splits):
        g[s, off["W_q"]:off["W_q"] + R * 2 * Hh] = torch.randn(R * 2 * Hh, generator=gen)
        g[s, off["b_q"]:off["b_q"] + R] = torch.randn(R, generator=gen)
    lib = _lib.lib()
    scratch = torch.empty(lib.rb200_dueling_scratch_floats(Hh, splits), device="cuda")
    outs = []
    for _ in range(2):
        gd = g.cuda()
        _lib.check(lib.rb200_dueling_unfold(gd.data_ptr(), stride, splits, A, N, Hh, off["W_q"],
                                            off["b_q"], off["W_adv"], off["b_adv"], off["w_val"],
                                            off["b_val"], scratch.data_ptr(), _lib.cur_stream()),
                   "rb200_dueling_unfold")
        torch.cuda.synchronize()
        outs.append(gd.cpu())
    assert torch.equal(outs[0], outs[1])
    got = outs[0]
    written = torch.zeros(stride, dtype=torch.bool)
    for k, n in sizes:
        written[off[k]:off[k] + n] = True
    assert bool((got[:, ~written] == SENT).all()), "a gap between the regions was written"
    zeros = [torch.zeros(R, Hh), torch.zeros(R), torch.zeros(N, Hh), torch.zeros(N)]
    for s in range(splits):
        seg = lambda k, n: got[s, off[k]:off[k] + n]  # noqa: E731
        assert bool((seg("W_q", R * 2 * Hh) == 0).all()) and bool((seg("b_q", R) == 0).all())
        want = H.dueling_unfold(*zeros, g[s, off["W_q"]:off["W_q"] + R * 2 * Hh].view(R, 2 * Hh),
                                g[s, off["b_q"]:off["b_q"] + R], A, N)
        for (k, n), w in zip(sizes[2:], want):
            _close(seg(k, n), w.reshape(-1), (s, k))


# ---------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("kind", ["qrdqn", "c51"])
def test_distributional_trainer_on_dueling_network_two_updates(kind):
    """Two consecutive train_batch calls of C51Trainer / QRDQNTrainer on a DuelingQNetwork with
    atoms: each update's q_network_grads() against fp64 autograd of the dueling head and the
    loss at that update's starting parameters (a stale folded layer on the second update, or
    a gradient left on the folded layer, fails here)."""
    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import CategoricalDQN, DuelingQNetwork
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import C51Trainer, QRDQNTrainer

    from oracle import td_oracle as O

    S, A, N, B = 10, 6, 11, 96
    qmin, qmax = -4.0, 6.0
    torch.manual_seed(21)
    net = DuelingQNetwork.make_fully_connected(S, A, [32, 24], ["relu", "relu"], num_atoms=N)
    rl = RLParameters(gamma=0.9, target_update_rate=0.1, maxq_learning=True)
    common = dict(actions=[str(i) for i in range(A)], rl=rl, double_q_learning=True,
                  minibatch_size=B, num_atoms=N, optimizer=Optimizer__Union.default(lr=0.05))
    if kind == "c51":
        q = CategoricalDQN(net, qmin=qmin, qmax=qmax, num_atoms=N)
        qt = q.get_target_network()
        t = C51Trainer(q.cuda(), qt.cuda(), qmin=qmin, qmax=qmax, **common).cuda()
        qnet, qtnet = q.distributional_network, qt.distributional_network
    else:
        qt = net.get_target_network()
        t = QRDQNTrainer(net, qt, evaluation=EvaluationParameters(calc_cpe_in_training=False),
                         **common).cuda()
        qnet, qtnet = t.q_network, t.q_network_target
    gen = torch.Generator().manual_seed(22)
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen) * 2, action=_onehot(B, A, gen),
             next_action=_onehot(B, A, gen),
             not_terminal=(torch.rand(B, 1, generator=gen) > 0.2).float(),
             possible_next_actions_mask=torch.ones(B, A))
    batch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(b["state"].cuda()), next_state=rlt.FeatureData(b["next_state"].cuda()),
        reward=b["reward"].cuda(), time_diff=torch.ones(B, 1, device="cuda"), step=None,
        not_terminal=b["not_terminal"].cuda(), action=b["action"].cuda(),
        next_action=b["next_action"].cuda(), possible_actions_mask=torch.ones(B, A, device="cuda"),
        possible_next_actions_mask=torch.ones(B, A, device="cuda"), extras=rlt.ExtraData())
    b64 = {k: v.double() for k, v in b.items()}

    for it in range(2):
        qo, qto = _oracle_dueling(qnet), _oracle_dueling(qtnet)
        params = O.net_params(qo)
        for p in params:
            p.requires_grad_(True)
        old = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)
        try:
            if kind == "c51":
                loss = O.c51_loss(qo, qto, b64, gamma=0.9, num_atoms=N, qmin=qmin, qmax=qmax)
            else:
                loss, _ = O.qrdqn_loss(qo, qto, b64, gamma=0.9, num_atoms=N)
        finally:
            torch.set_default_dtype(old)
        want = torch.autograd.grad(loss, params)
        got_loss = float(t.train_batch(batch, it))
        got = t.q_network_grads()
        assert len(got) == len(want)
        want_loss = float(loss.detach())
        assert abs(got_loss - want_loss) <= TOL * max(1.0, abs(want_loss)), (it, got_loss, want_loss)
        for i, (x, w) in enumerate(zip(got, want)):
            assert G.rel_err(x, w) < TOL, (it, i, G.rel_err(x, w))


def _oracle_dueling(module):
    """td_oracle's dueling network (float64) from a DuelingQNetwork's current parameters, in
    the registration order shared / advantage / value (dueling_q_network.py:48-90)."""
    ps = [p.detach().cpu().double() for p in module.parameters()]
    n_shared = len(ps) - 8  # each head: [E -> E/2 -> out], two Linear layers
    half = lambda lst: {"W": lst[0::2], "b": lst[1::2]}  # noqa: E731
    shared = half(ps[:n_shared])
    return {"kind": "dueling",
            "shared": {**shared, "act": ["relu"] * (len(shared["W"]) - 1) + ["linear"]},
            "adv": {**half(ps[n_shared:n_shared + 4]), "act": ["relu", "linear"]},
            "val": {**half(ps[n_shared + 4:]), "act": ["relu", "linear"]}}
