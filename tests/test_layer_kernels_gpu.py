"""The shared layer primitives and the optimizer under every trainer, called through the C ABI
and compared with plain references at the shapes where tiled kernels go wrong.

* rb200_mlp_forward / rb200_mlp_backward / rb200_linear_backward_dx (row-tile path) against an
  fp64 chain computed from exactly the fp32 inputs the kernel received, in every row-tile
  configuration (RB200_FORCE_CFG) and at the 256-column chunk and k-chunk edges.
* rb200_mlp_wgrad (the mma.sync kernel) slab by slab against fp64 dZ^T.A, with the
  gradient partials prefilled with NaN so an unwritten (empty) slab cannot pass.
* rb200_grad_reduce bit for bit against a sequential fp32 sum in slab order.
* rb200_adam_soft_update / FusedAdam against torch.optim.Adam(foreach=False) on the CPU, and
  the Polyak updates against SoftUpdate's formula.

Random weights are scaled by 1/sqrt(fan_in), so every output row and column is O(1) and an
error confined to a ragged tail cannot hide under the tensor's maximum.  Measured errors are
appended to $RB200_TEST_RECORD_DIR/test_measurements.jsonl when that directory exists.
"""
import math

import numpy as np
import pytest
import torch

from reagent_b200 import _lib
from tests import golden_util as G
from tests.builders import _record
from tests.kernel_util import (BETAS, CFGS, E_SMEM, EPS, GRAD_SCALE, LR, NAN, NUM_SMS, TAU,
                               TOL, _cfg_id, _fits, _padded, _seq_sum, _set_cfg, _tol)

pytestmark = pytest.mark.gpu

ACTS = ["linear", "relu", "tanh", "leaky_relu", "sigmoid", "softplus"]


def _lib_():
    return _lib.lib()


def _stream():
    return _lib.cur_stream()


# ------------------------------------------------------------------------------------------
# networks in the arena layout (models/arena.py) and their fp64 references
# ------------------------------------------------------------------------------------------
class Net:
    def __init__(self, dims, acts, seed=0, w_shift=0):
        from reagent_b200.models.arena import ParamArena

        self.dims, self.acts = list(dims), list(acts)
        ar = ParamArena(dims, [_lib.ACT[a] for a in acts])
        self.w_off = [o + w_shift for o in ar.w_off]
        self.b_off = [o + w_shift for o in ar.b_off]
        self.n = ar.n + w_shift
        g = torch.Generator().manual_seed(seed)
        flat = torch.full((self.n,), NAN)
        self.W, self.b = [], []
        for l in range(len(acts)):
            K, N = dims[l], dims[l + 1]
            W = torch.randn(N, K, generator=g) / math.sqrt(K)
            b = 0.5 * torch.randn(N, generator=g)
            flat[self.w_off[l]:self.w_off[l] + N * K] = W.reshape(-1)
            flat[self.b_off[l]:self.b_off[l] + N] = b
            self.W.append(W)
            self.b.append(b)
        self.flat = flat.cuda()

    def desc(self):
        d = _lib.MlpT()
        d.n_layers = len(self.acts)
        for i, v in enumerate(self.dims):
            d.dims[i] = v
        for i, a in enumerate(self.acts):
            d.act[i] = _lib.ACT[a]
            d.w_off[i] = self.w_off[i]
            d.b_off[i] = self.b_off[i]
        d.params = self.flat.data_ptr()
        d.n_params = self.n
        return d


def _act64(z, act):
    if act == "relu":
        return torch.relu(z)
    if act == "tanh":
        return torch.tanh(z)
    if act == "leaky_relu":
        return torch.nn.functional.leaky_relu(z, 0.01)
    if act == "sigmoid":
        return torch.sigmoid(z)
    if act == "softplus":
        return torch.nn.functional.softplus(z)
    return z


def _dact64(h, act):
    """act'(z) through the activation's output h (as the kernels evaluate it)."""
    if act == "relu":
        return (h > 0).double()
    if act == "tanh":
        return 1.0 - h * h
    if act == "leaky_relu":
        return torch.where(h > 0, 1.0, 0.01).double()
    if act == "sigmoid":
        return h * (1.0 - h)
    if act == "softplus":
        return 1.0 - torch.exp(-h)
    return torch.ones_like(h)


def _forward64(net, x):
    hs, h = [], x.double()
    for l, a in enumerate(net.acts):
        h = _act64(h @ net.W[l].double().T + net.b[l].double(), a)
        hs.append(h)
    return hs  # hs[-1] is the output


def _ws(hidden=(), dz=()):
    ws = _lib.NetWsT()
    for i, t in enumerate(hidden):
        ws.hidden[i] = None if t is None else t.data_ptr()
    for i, t in enumerate(dz):
        ws.dz[i] = None if t is None else t.data_ptr()
    return ws


# ------------------------------------------------------------------------------------------
# (a) rb200_mlp_forward
# ------------------------------------------------------------------------------------------
FWD_NETS = [
    ([1, 255, 3], ["tanh", "linear"]),                                   # K = 1
    ([3, 256, 257, 31], ["relu", "sigmoid", "linear"]),                  # 256 / 257 columns
    ([31, 513, 5], ["softplus", "leaky_relu"]),                          # three column chunks
    ([32, 257], ["tanh"]),                                               # one layer
    ([33, 64, 48, 40, 36, 33, 32, 31, 7], ACTS + ["relu", "linear"]),    # 8 layers, every act
    ([600, 320, 4], ["relu", "linear"]),                                 # first fit (512, 16)
    ([1000, 800, 4], ["tanh", "linear"]),                                # only (256, 16) fits
]


def _run_forward(net, x0, x1, batch, offset):
    L = len(net.acts)
    out = _padded((batch, net.dims[-1]), offset)
    hid = [_padded((batch, net.dims[l + 1]), offset) for l in range(L - 1)]
    ws = _ws(hidden=hid)
    d = net.desc()
    d1 = 0 if x1 is None else x1.shape[1]
    rc = _lib_().rb200_mlp_forward(d, x0.data_ptr(), x0.shape[1], _lib.ptr(x1), d1, batch,
                                   out.data_ptr(), ws, _stream())
    torch.cuda.synchronize()
    return rc, out, hid


@pytest.mark.parametrize("batch", [1, 15, 16, 17, 33, 2113])
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_mlp_forward_matches_fp64(monkeypatch, cfg, batch):
    _set_cfg(monkeypatch, cfg)
    worst = 0.0
    for i, (dims, acts) in enumerate(FWD_NETS):
        net = Net(dims, acts, seed=i)
        g = torch.Generator().manual_seed(100 + i)
        x = torch.randn(batch, dims[0], generator=g)
        offset = (i + batch) % 2  # half the cases unaligned
        x_dev = _padded(x.shape, offset)
        x_dev.copy_(x)
        hmax = max(dims[1:-1], default=0)
        fits = _fits(cfg, batch, dims[0], hmax, 1, 2, ((dims[-1] + 3) & ~3) + 4)
        rc, out, hid = _run_forward(net, x_dev, None, batch, offset)
        if not fits:
            assert rc == E_SMEM, (dims, rc)
            assert torch.isnan(out).all(), "a refused forward must not launch"
            continue
        assert rc == 0, (dims, _lib_().rb200_last_error())
        ref = _forward64(net, x)
        tol = _tol(max(dims[:-1]))
        for l in range(len(acts) - 1):
            e = G.rel_err(hid[l], ref[l])
            worst = max(worst, e)
            assert e < tol, (dims, "hidden", l, e)
        e = G.rel_err(out, ref[-1])
        worst = max(worst, e)
        assert e < tol, (dims, "out", e)
    _record("mlp_forward", cfg=_cfg_id(cfg), batch=batch, max_rel_err=worst)


@pytest.mark.parametrize("act", ACTS)
def test_mlp_forward_each_activation_and_concat(act):
    """cat(in0, in1) staging with d0 % 4 != 0 and unaligned inputs, for each activation."""
    worst = 0.0
    for batch in (17, 2113):
        for d0, d1, off in ((3, 5, 1), (6, 7, 0), (1, 1, 1)):
            net = Net([d0 + d1, 257, 9], [act, act], seed=d0 * 7 + d1)
            g = torch.Generator().manual_seed(d0)
            x0, x1 = torch.randn(batch, d0, generator=g), torch.randn(batch, d1, generator=g)
            x0d, x1d = _padded(x0.shape, off), _padded(x1.shape, 1 - off)
            x0d.copy_(x0)
            x1d.copy_(x1)
            rc, out, hid = _run_forward(net, x0d, x1d, batch, off)
            assert rc == 0, _lib_().rb200_last_error()
            ref = _forward64(net, torch.cat([x0, x1], 1))
            e = max(G.rel_err(out, ref[-1]), G.rel_err(hid[0], ref[0]))
            worst = max(worst, e)
            assert e < TOL, (act, batch, d0, d1, e)
    _record("mlp_forward_concat", act=act, max_rel_err=worst)


def test_mlp_forward_refuses_shapes_without_a_tile():
    lib = _lib_()
    x = torch.randn(4, 8192, device="cuda")
    net = Net([8192, 4], ["linear"])
    out = _padded((4, 4))
    rc = lib.rb200_mlp_forward(net.desc(), x.data_ptr(), 8192, None, 0, 4, out.data_ptr(), None,
                               _stream())
    assert rc == E_SMEM
    assert b"shared memory" in lib.rb200_last_error()
    net = Net([8, 1025], ["linear"])
    out = _padded((4, 1025))
    rc = lib.rb200_mlp_forward(net.desc(), x.data_ptr(), 8, None, 0, 4, out.data_ptr(), None,
                               _stream())
    assert rc == E_SMEM
    assert b"1025" in lib.rb200_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


# ------------------------------------------------------------------------------------------
# (b) rb200_mlp_backward and the row-tile rb200_linear_backward_dx
# ------------------------------------------------------------------------------------------
BWD_NETS = [
    ([5, 255, 3], ["tanh", "linear"]),
    ([3, 256, 257, 31], ["sigmoid", "softplus", "linear"]),
    ([31, 513, 33, 5], ["leaky_relu", "relu", "linear"]),
    ([33, 64, 48, 40, 36, 33, 32, 31, 7], ACTS + ["tanh", "linear"]),
    ([8, 800, 1], ["softplus", "linear"]),
]


@pytest.mark.parametrize("batch", [1, 15, 16, 17, 33, 2113])
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_mlp_backward_matches_fp64(monkeypatch, cfg, batch):
    _set_cfg(monkeypatch, cfg)
    worst = 0.0
    for i, (dims, acts) in enumerate(BWD_NETS):
        L = len(acts)
        net = Net(dims, acts, seed=10 + i)
        g = torch.Generator().manual_seed(200 + i)
        # the saved activations are the fp64 forward cast to fp32: act' sees the same h here
        h32 = [h.float() for h in _forward64(net, torch.randn(batch, dims[0], generator=g))[:-1]]
        dz_last = torch.randn(batch, dims[-1], generator=g)
        offset = i % 2
        hid = []
        for h in h32:
            t = _padded(h.shape, offset)
            t.copy_(h)
            hid.append(t)
        dz = [_padded((batch, dims[l + 1]), offset) for l in range(L - 1)] + [None]
        dzl = _padded(dz_last.shape, offset)
        dzl.copy_(dz_last)
        fits = _fits(cfg, batch, 4, max(dims[1:-1]), 0, 3, ((dims[-1] + 3) & ~3) + 4)
        rc = _lib_().rb200_mlp_backward(net.desc(), dzl.data_ptr(), batch, _ws(hid, dz), _stream())
        torch.cuda.synchronize()
        if not fits:
            assert rc == E_SMEM
            assert all(torch.isnan(t).all() for t in dz[:-1])
            continue
        assert rc == 0, _lib_().rb200_last_error()
        ref = dz_last.double()
        for l in range(L - 1, 0, -1):
            ref = (ref @ net.W[l].double()) * _dact64(h32[l - 1].double(), acts[l - 1])
            e = G.rel_err(dz[l - 1], ref)
            worst = max(worst, e)
            assert e < _tol(max(dims[1:])), (dims, l - 1, e)
    _record("mlp_backward", cfg=_cfg_id(cfg), batch=batch, max_rel_err=worst)


LINBWD_SHAPES = [(1, 33), (3, 1), (31, 513), (32, 255), (33, 1025), (255, 64), (256, 257),
                 (257, 7), (513, 100), (1024, 31)]   # (K, N): out [B, K] = dz [B, N] . W [N, K]


@pytest.mark.parametrize("batch", [1, 15, 16, 17, 33, 2113])
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_linear_backward_dx_matches_fp64(monkeypatch, cfg, batch):
    _set_cfg(monkeypatch, cfg)
    worst = 0.0
    for i, (K, N) in enumerate(LINBWD_SHAPES):
        act = ACTS[i % len(ACTS)]
        g = torch.Generator().manual_seed(300 + i)
        W = torch.randn(N, K, generator=g) / math.sqrt(N)
        dz = torch.randn(batch, N, generator=g)
        h = _act64(torch.randn(batch, K, generator=g).double(), act).float()
        offset = i % 2
        Wd, dzd, hd = _padded(W.shape, offset), _padded(dz.shape, 1 - offset), _padded(h.shape, offset)
        Wd.copy_(W)
        dzd.copy_(dz)
        hd.copy_(h)
        fits = _fits(cfg, batch, 512, 4, 1, 0, 2 * (((K + 3) & ~3) + 4))
        for use_h in (True, False):
            out = _padded((batch, K), offset)
            rc = _lib_().rb200_linear_backward_dx(Wd.data_ptr(), K, N, dzd.data_ptr(),
                                                  hd.data_ptr() if use_h else None,
                                                  _lib.ACT[act], batch, out.data_ptr(), _stream())
            torch.cuda.synchronize()
            if not fits:
                assert rc == E_SMEM
                assert torch.isnan(out).all()
                continue
            assert rc == 0, _lib_().rb200_last_error()
            ref = dz.double() @ W.double()
            if use_h:
                ref = ref * _dact64(h.double(), act)
            e = G.rel_err(out, ref)
            worst = max(worst, e)
            assert e < TOL, (K, N, act, use_h, e)
    _record("linear_backward_dx", cfg=_cfg_id(cfg), batch=batch, max_rel_err=worst)


# ------------------------------------------------------------------------------------------
# (c) rb200_mlp_wgrad and rb200_grad_reduce
# ------------------------------------------------------------------------------------------
# every layer sits on an edge of the kernel's 64x64 tiles
WGRAD_NETS = [
    [65, 63, 64, 129, 257, 127, 255, 128, 256],
    [1, 3, 1],
]


def _rows_per_split(batch, splits):
    return -(-(-(-batch // splits)) // 32) * 32


def _wgrad_inputs(net, batch, seed, offset=0):
    g = torch.Generator().manual_seed(seed)
    L = len(net.acts)
    acts = [torch.randn(batch, net.dims[l], generator=g) for l in range(L)]
    dZs = [torch.randn(batch, net.dims[l + 1], generator=g) for l in range(L)]
    dev = []
    for t in acts + dZs:
        d = _padded(t.shape, offset)
        d.copy_(t)
        dev.append(d)
    return acts, dZs, dev[:L], dev[L:]


@pytest.mark.parametrize("kernel", ["mma_sync"])
@pytest.mark.parametrize("batch", [1, 31, 100, 257, 4096])
def test_mlp_wgrad_slabs_match_fp64(kernel, batch):
    lib = _lib_()
    worst = 0.0
    for ni, dims in enumerate(WGRAD_NETS):
        net = Net(dims, ["relu"] * (len(dims) - 2) + ["linear"], seed=ni)
        acts, dZs, acts_d, dZs_d = _wgrad_inputs(net, batch, 400 + ni)
        # layer l's input activation is hidden[l-1]: feed the random activations through ws
        ws = _ws(hidden=acts_d[1:], dz=dZs_d)
        d = net.desc()
        split_set = sorted({1, 3, 8, lib.rb200_wgrad_splits(batch), 64})
        for splits in split_set:
            gpart = torch.full((splits, net.n), NAN, device="cuda")
            rc = lib.rb200_mlp_wgrad(d, acts_d[0].data_ptr(), batch, ws, gpart.data_ptr(), splits,
                                     _stream())
            assert rc == 0, lib.rb200_last_error()
            torch.cuda.synchronize()
            worst = max(worst, _check_wgrad_layers(net, acts, dZs, batch, splits, gpart,
                                                   (dims, splits)))
    _record("mlp_wgrad", kernel=kernel, batch=batch, max_rel_err=worst)


def _check_wgrad_layers(net, acts, dZs, batch, splits, gpart, what):
    rps = _rows_per_split(batch, splits)
    gp = gpart.cpu().double()
    worst = 0.0
    for l in range(len(net.acts)):
        K, N = net.dims[l], net.dims[l + 1]
        a, z = acts[l].double(), dZs[l].double()
        wsl = gp[:, net.w_off[l]:net.w_off[l] + N * K].reshape(splits, N, K)
        bsl = gp[:, net.b_off[l]:net.b_off[l] + N]
        assert torch.isfinite(wsl).all() and torch.isfinite(bsl).all(), (what, l, "unwritten")
        for s in range(splits):
            r0, r1 = min(batch, s * rps), min(batch, (s + 1) * rps)
            if r0 == r1:
                assert (wsl[s] == 0).all() and (bsl[s] == 0).all(), (what, l, s, "empty slab")
                continue
            ew = G.rel_err(wsl[s], z[r0:r1].T @ a[r0:r1])
            eb = G.rel_err(bsl[s], z[r0:r1].sum(0))
            worst = max(worst, ew, eb)
            assert ew < _tol(r1 - r0) and eb < _tol(r1 - r0), (what, l, s, ew, eb)
        ew = G.rel_err(wsl.sum(0), z.T @ a)
        eb = G.rel_err(bsl.sum(0), z.sum(0))
        worst = max(worst, ew, eb)
        assert ew < _tol(min(rps, batch)) and eb < _tol(min(rps, batch)), (what, l, ew, eb)
    return worst


@pytest.mark.parametrize("kernel", ["mma_sync"])
def test_mlp_wgrad_odd_offsets_and_unaligned_inputs(kernel):
    """A hand-built descriptor whose weights start at odd arena offsets over activations that
    are not 16-byte aligned (scalar staging)."""
    lib = _lib_()
    worst = 0.0
    for batch in (100, 257):
        net = Net([64, 128, 256, 129], ["relu", "tanh", "linear"], seed=7, w_shift=1)
        assert all(o % 2 == 1 for o in net.w_off)
        acts, dZs, acts_d, dZs_d = _wgrad_inputs(net, batch, 500, offset=1)
        ws = _ws(hidden=acts_d[1:], dz=dZs_d)
        for splits in (1, 3, 8):
            gpart = torch.full((splits, net.n), NAN, device="cuda")
            rc = lib.rb200_mlp_wgrad(net.desc(), acts_d[0].data_ptr(), batch, ws,
                                     gpart.data_ptr(), splits, _stream())
            assert rc == 0, lib.rb200_last_error()
            torch.cuda.synchronize()
            worst = max(worst, _check_wgrad_layers(net, acts, dZs, batch, splits, gpart,
                                                   ("odd w_off", batch, splits)))
    _record("mlp_wgrad_odd_offsets", kernel=kernel, max_rel_err=worst)


@pytest.mark.parametrize("n", [1, 255, 257, NUM_SMS * 8 * 256 + 5])
@pytest.mark.parametrize("splits", [1, 3, 8, 64])
def test_grad_reduce_bit_identical_to_sequential_fp32(n, splits):
    g = torch.Generator().manual_seed(n + splits)
    parts = torch.randn(splits, n, generator=g) * torch.logspace(-3, 3, splits).view(-1, 1)
    out = _padded((n,))
    parts_dev = parts.cuda()
    rc = _lib_().rb200_grad_reduce(parts_dev.data_ptr(), splits, n, out.data_ptr(), _stream())
    assert rc == 0
    p = parts.numpy()
    ref = p[0].copy()
    for s in range(1, splits):
        ref = (ref + p[s]).astype(np.float32)
    assert np.array_equal(out.cpu().numpy().view(np.int32), ref.view(np.int32))


# ------------------------------------------------------------------------------------------
# (d) rb200_adam_soft_update, rb200_soft_update, FusedAdam against torch on the CPU
# ------------------------------------------------------------------------------------------


def _adam_inputs(opt, ref_p):
    """(exp_avg_sq before the step, gradient after weight decay) as torch.optim.Adam sees them;
    call after setting ref_p.grad and before opt.step()."""
    st = opt.state.get(ref_p, {})
    v_prev = st["exp_avg_sq"].clone() if "exp_avg_sq" in st else torch.zeros_like(ref_p)
    g = ref_p.grad.add(ref_p.detach(), alpha=opt.param_groups[0]["weight_decay"])
    return v_prev, g


def _check_adam_step(p_dev, m_dev, v_dev, ref_p, opt, p_prev, v_prev, g, what):
    """One step of the kernel against torch.optim.Adam's single-tensor CPU path from identical
    state.  Two roundings are allowed to differ, and both are checked exactly instead:

    * exp_avg_sq.  The kernel rounds addcmul's product and sum separately:
      v*b2 + ((1-b2)*g)*g.  ATen's AVX2 / AVX-512 builds contract the last multiply-add into an
      fma, which can land 1 ulp away.  So exp_avg_sq must equal that separately rounded rule bit
      for bit, and be within 1 ulp of torch's.
    * the square root.  torch.sqrt on the CPU comes from the host's vector math library, which
      can miss the correctly rounded root by an ulp.  The kernel computes the correctly rounded
      root (__fsqrt_rn).

    exp_avg must equal torch's bit for bit.  The parameters must equal torch's update rule,
    bit for bit and everywhere, when that rule uses the kernel's exp_avg_sq and the correctly
    rounded root: p + (-step_size * m) / (sqrt_rn(v) / sqrt(bc2) + eps).  Where neither
    rounding differs, that is torch's own result, and that is asserted too.  Afterwards torch's
    exp_avg_sq and parameters are copied back, so the next step starts from identical state.
    Returns (elements whose exp_avg_sq differs by 1 ulp, elements where torch's sqrt was not
    correctly rounded)."""
    st = opt.state[ref_p]
    grp = opt.param_groups[0]
    b2 = grp["betas"][1]
    m_ref, v_ref = st["exp_avg"], st["exp_avg_sq"]
    assert torch.equal(m_dev.cpu(), m_ref), (what, "exp_avg")
    v_got = v_dev.cpu()
    v_rule = v_prev * b2 + ((1 - b2) * g) * g
    assert torch.equal(v_got, v_rule), (what, "exp_avg_sq vs separately rounded rule")
    v_ulps = (v_got.view(torch.int32).long() - v_ref.view(torch.int32).long()).abs()
    assert int(v_ulps.max()) <= 1, (what, "exp_avg_sq vs torch", int(v_ulps.max()))
    p_got, p_ref = p_dev.cpu(), ref_p.detach()
    cr = torch.from_numpy(np.sqrt(v_got.numpy().astype(np.float64)).astype(np.float32))
    t = float(st["step"])
    step_size = grp["lr"] / (1 - grp["betas"][0] ** t)
    bc2_sqrt = (1 - b2 ** t) ** 0.5
    p_rule = p_prev + (-step_size * m_ref) / (cr / bc2_sqrt + grp["eps"])
    assert torch.equal(p_got, p_rule), (what, "params vs update rule", int((p_got != p_rule).sum()))
    inexact = v_ref.sqrt() != torch.from_numpy(
        np.sqrt(v_ref.numpy().astype(np.float64)).astype(np.float32))
    same_path = (v_ulps == 0) & ~inexact
    assert torch.equal(p_got[same_path], p_ref[same_path]), (what, "params vs torch")
    v_dev.copy_(v_ref)
    p_dev.copy_(p_ref)
    return int((v_ulps != 0).sum()), int(inexact.sum())


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("splits", [1, 7, 8, 9, 64])
@pytest.mark.parametrize("n", [1, 255, 257, NUM_SMS * 4 * 256 + 3])
def test_adam_soft_update_matches_torch_adam(n, splits, weight_decay):
    lib = _lib_()
    g = torch.Generator().manual_seed(n * 131 + splits)
    p0 = torch.randn(n, generator=g)
    tgt0 = torch.randn(n, generator=g)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref_p], lr=LR, betas=BETAS, eps=EPS, weight_decay=weight_decay,
                           foreach=False)
    p_dev, tgt = p0.cuda(), tgt0.cuda()
    m_dev, v_dev = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    exp_out = _padded((n,))
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    v_off = inexact = 0
    for it in range(50):
        parts = torch.randn(splits, n, generator=g) * 0.1
        parts_dev = parts.cuda()
        a = _lib.AdamArgsT()
        a.params, a.grad, a.splits, a.n = p_dev.data_ptr(), parts_dev.data_ptr(), splits, n
        a.exp_avg, a.exp_avg_sq = m_dev.data_ptr(), v_dev.data_ptr()
        a.step, a.block_counter = step.data_ptr(), counter.data_ptr()
        a.lr, a.beta1, a.beta2, a.eps, a.weight_decay = LR, BETAS[0], BETAS[1], EPS, weight_decay
        a.grad_scale = GRAD_SCALE
        a.target, a.tau, a.one_minus_tau = tgt.data_ptr(), TAU, float(1.0 - TAU)
        a.exp_out = exp_out.data_ptr()
        a.dp_world = 1
        tgt_before = tgt.cpu()
        assert lib.rb200_adam_soft_update(a, _stream()) == 0, lib.rb200_last_error()
        torch.cuda.synchronize()
        p_prev = ref_p.detach().clone()
        ref_p.grad = _seq_sum(parts) * GRAD_SCALE
        v_prev, g_eff = _adam_inputs(opt, ref_p)
        opt.step()
        p_new = p_dev.cpu()
        # the fused Polyak update reads the kernel's own new parameters
        assert torch.equal(tgt.cpu(), TAU * p_new + (1.0 - TAU) * tgt_before), (n, it, "target")
        e = exp_out.cpu()
        ulps = (e.view(torch.int32).long() - torch.exp(p_new).view(torch.int32).long()).abs()
        assert int(ulps.max()) <= 2, (n, it, "exp_out")
        dv, ds = _check_adam_step(p_dev, m_dev, v_dev, ref_p, opt, p_prev, v_prev, g_eff,
                                  (n, splits, it))
        v_off, inexact = v_off + dv, inexact + ds
        assert int(step.item()) == it + 1
    _record("adam_vs_torch", n=n, splits=splits, weight_decay=weight_decay, steps=50,
            exp_avg_sq_1ulp_elements=v_off, inexact_sqrt_elements=inexact)


@pytest.mark.parametrize("n", [1, 257, NUM_SMS * 4 * 256 + 3])
def test_soft_update_bit_identical_to_softupdate_formula(n):
    lib = _lib_()
    g = torch.Generator().manual_seed(n)
    src, tgt0 = torch.randn(n, generator=g), torch.randn(n, generator=g)
    src_dev = src.cuda()
    for tau in (0.3, 1e-3, 0.999):
        tgt = tgt0.cuda()
        rc = lib.rb200_soft_update(tgt.data_ptr(), src_dev.data_ptr(), n, tau, float(1.0 - tau),
                                   _stream())
        assert rc == 0
        assert torch.equal(tgt.cpu(), tau * src + (1.0 - tau) * tgt0), (n, tau)
    # target is source: SoftUpdate skips it
    t = tgt0.cuda()
    assert lib.rb200_soft_update(t.data_ptr(), t.data_ptr(), n, 0.3, 0.7, _stream()) == 0
    assert torch.equal(t.cpu(), tgt0)


def test_fused_adam_state_dict_round_trip_with_torch_adam():
    """10 FusedAdam steps; its state_dict resumes a CPU torch.optim.Adam, and that one's
    state_dict resumes a fresh FusedAdam.  Then 10 more steps on all three with the same
    gradients: the two FusedAdams stay bit-identical, and torch matches them step by step
    (with the two named roundings of _check_adam_step)."""
    from reagent_b200.models import FullyConnectedNetwork
    from reagent_b200.optimizer import FusedAdam

    torch.manual_seed(0)
    kw = dict(lr=LR, betas=BETAS, eps=EPS, weight_decay=1e-2)
    net = FullyConnectedNetwork([7, 33, 5], ["tanh", "linear"]).cuda()
    f1 = FusedAdam(net.parameters(), **kw)
    ar = f1.arena
    g = torch.Generator().manual_seed(3)
    grads = [torch.randn(3, ar.n, generator=g) * 0.1 for _ in range(20)]
    for k in range(10):
        f1.fused_step(grad=grads[k].cuda(), grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()

    cpu_net = FullyConnectedNetwork([7, 33, 5], ["tanh", "linear"])
    cpu_net.load_state_dict({k: v.cpu() for k, v in net.state_dict().items()})
    t2 = torch.optim.Adam(cpu_net.parameters(), foreach=False, **kw)
    t2.load_state_dict(f1.state_dict())
    net3 = FullyConnectedNetwork([7, 33, 5], ["tanh", "linear"]).cuda()
    net3.load_state_dict(net.state_dict())
    f3 = FusedAdam(net3.parameters())
    f3.load_state_dict(t2.state_dict())
    assert f3.num_steps == 10

    params = list(cpu_net.parameters())
    v_off = inexact = 0
    for k in range(10, 20):
        gd = grads[k].cuda()
        f1.fused_step(grad=gd, grad_scale=GRAD_SCALE)
        f3.fused_step(grad=gd, grad_scale=GRAD_SCALE)
        flat_g = _seq_sum(grads[k]) * GRAD_SCALE
        prev = [p.detach().clone() for p in params]
        for l in range(2):
            params[2 * l].grad = ar.weight_view(flat_g, l).clone()
            params[2 * l + 1].grad = ar.bias_view(flat_g, l).clone()
        before = [_adam_inputs(t2, p) for p in params]
        t2.step()
        torch.cuda.synchronize()
        for l in range(2):
            for j, view in enumerate((ar.weight_view, ar.bias_view)):
                # the arena's alignment padding is not state: compare the parameters only
                for t1, t3 in ((f1.arena.flat, f3.arena.flat), (f1.exp_avg, f3.exp_avg),
                               (f1.exp_avg_sq, f3.exp_avg_sq)):
                    assert torch.equal(view(t1, l), view(t3, l)), (k, l, j)
                p = params[2 * l + j]
                dv, ds = _check_adam_step(view(f1.arena.flat, l), view(f1.exp_avg, l),
                                          view(f1.exp_avg_sq, l), p, t2, prev[2 * l + j],
                                          *before[2 * l + j], ("round trip", k, l, j))
                v_off, inexact = v_off + dv, inexact + ds
        # keep f3 on the same (torch-synchronised) state as f1
        f3.arena.flat.copy_(f1.arena.flat)
        f3.exp_avg_sq.copy_(f1.exp_avg_sq)
    assert f1.num_steps == f3.num_steps == 20
    _record("adam_state_dict_round_trip", exp_avg_sq_1ulp_elements=v_off,
            inexact_sqrt_elements=inexact)
