"""Constants and launch helpers of the kernel-level tests (the layer, Adam, loss-reduction,
loss-head and actor-critic kernels) that more than one test module uses."""
import ctypes as C

import numpy as np
import torch

from reagent_b200 import _lib

NAN = float("nan")
NUM_SMS = 132
E_SMEM = -3         # RB200_E_SMEM: no row tile fits in shared memory
TOL = 1e-5          # the project's parity bar


def _tol(length):
    """Bound for a contraction of `length` terms run as one chain of MMAs into an fp32
    accumulator.  The project's 1e-5 holds up to 256 terms; beyond that the accumulator's own
    rounding (NVIDIA's tensor cores do not round the fp32 accumulation to nearest) adds up with
    the number of k steps, so the bound grows linearly with the length.  Measured on an H100:
    2.2e-5 for the forward at K = 1000, 3.3e-5 for one 4096-row weight-gradient slab."""
    return TOL * max(1.0, length / 256)


# pick_rows_cfg's four instances (threads, k-chunk) and the default choice
CFGS = [None, (512, 32), (512, 16), (256, 32), (256, 16)]
SMEM_FLOATS = 227 * 1024 // 4


def _cfg_id(c):
    return "default" if c is None else f"{c[0]}x{c[1]}"


def _set_cfg(monkeypatch, cfg):
    """Force the row-tile kernels onto one (threads, k-chunk) instance (None: their own
    choice).  pick_rows_cfg reads RB200_FORCE_CFG at every launch."""
    if cfg is None:
        monkeypatch.delenv("RB200_FORCE_CFG", raising=False)
    else:
        monkeypatch.setenv("RB200_FORCE_CFG", f"{cfg[0]},{cfg[1]}")


def _fits(cfg, batch, din, hmax, n_in, n_h, extra_per_row):
    """Mirror of pick_rows_cfg (csrc/rb200_rows.cuh): does the forced (or any) tile fit?"""
    return _pick(cfg, batch, din, hmax, n_in, n_h, extra_per_row) is not None


def _pick(cfg, batch, din, hmax, n_in, n_h, extra_per_row):
    """Mirror of pick_rows_cfg: the (threads, k-chunk) it launches, or None when none fits."""
    r4 = lambda x: (x + 3) & ~3
    ld_in, ld_h = r4(din) + 4, r4(hmax if hmax > 0 else 4) + 4
    cands = [(512, 32), (512, 16), (256, 32), (256, 16)]
    for nt, kc in cands:
        R = (nt // 64) * 4
        if cfg is not None:
            if (nt, kc) != tuple(cfg):
                continue
        elif R == 32 and batch <= 16 * NUM_SMS:
            continue
        stage = max(256 * (kc + 4), kc * 264)
        if 2 * stage + R * (n_in * ld_in + n_h * ld_h + extra_per_row) <= SMEM_FLOATS:
            return (nt, kc)
    return None


def _r8(x):
    return (x + 7) & ~7


def _k2_image_bytes(N, K):
    """image_bytes (csrc/rb200_dqn_tc_layout.cuh): one [K/4][rows][4] block per 128-row tile,
    rows rounded up to 8 plus a 16-byte pad per k quad."""
    return sum((_r8(K) // 4) * (_r8(min(N - 128 * t, 128)) * 16 + 16)
               for t in range((N + 127) // 128))


def _k2_tc_bytes(dims, double_q, do_backward):
    """Mirror of rb200_dqn_tc_workspace_bytes (make_plan in csrc/rb200_dqn_tc.cu): the pack
    size tc_images gives for `dims`, or 0 when the wgmma TD kernel does not take the shape and
    K2 runs on the row-tile kernel.  `double_q` changes neither the images (the target's are
    always packed) nor the shared memory (the q(s') buffer is always reserved)."""
    del double_q
    L = len(dims) - 1
    if L < 1 or L > 8 or any(d > 4 * 128 or d > 32000 for d in dims[1:]):
        return 0
    if dims[0] > 32000 or dims[L] > 256:
        return 0
    fwd = sum(_k2_image_bytes(dims[l + 1], dims[l]) for l in range(L))
    bwd = sum(_k2_image_bytes(dims[l], dims[l + 1]) for l in range(1, L)) if do_backward else 0
    # shared memory: 3-stage ring of two 32-k chunk images of a full tile, two ping-pong
    # activation operands and the last layer's dZ (k quads of 64 rows hi/lo + 16 B), the three
    # q arrays [32][A + 1], action and mask rows, per-row scalars, the ring's mbarriers
    ring, lbo_b, R = 3 * 2 * 8 * (128 * 16 + 16), 64 * 16 + 16, 32
    A = dims[L]
    maxd = [8, 8, A]
    for i in range(L):
        maxd[i & 1] = max(maxd[i & 1], dims[i])
    a16 = lambda x: (x + 15) & ~15
    o = ring + sum(_r8(m) // 4 * lbo_b for m in maxd)
    o = a16(o + 3 * R * (A + 1) * 4)
    o = a16(o + (2 * R * A + 4 * R + 8) * 4)
    o = a16(o + 2 * 3 * 8)
    return 2 * fwd + bwd + 4096 if o <= 232448 else 0


def _padded(shape, offset=0, fill=NAN):
    """A CUDA fp32 tensor of `shape` starting `offset` floats into its allocation (offset 1:
    not 16-byte aligned, which sends the kernels down their scalar load / store paths)."""
    n = int(np.prod(shape))
    buf = torch.full((n + offset + 4,), fill, device="cuda")
    return buf[offset:offset + n].view(*shape)


LR, BETAS, EPS, GRAD_SCALE, TAU = 0.1, (0.5, 0.9), 1e-3, 0.5, 0.3


def _seq_sum(parts):
    s = parts[0].clone()
    for k in range(1, parts.shape[0]):
        s = s + parts[k]
    return s


def _call(fn, a):
    _lib.check(getattr(_lib.lib(), fn)(C.byref(a), _lib.cur_stream()), fn)
    torch.cuda.synchronize()


def _ws(n_partials, n_loss=1):
    return dict(partials=torch.full((n_partials,), float("nan"), device="cuda"),
                loss=torch.zeros(n_loss, device="cuda"),
                counter=torch.zeros(1, dtype=torch.int32, device="cuda"))


def _set_ws(a, ws):
    a.loss_partials, a.loss, a.tile_counter = (ws["partials"].data_ptr(), ws["loss"].data_ptr(),
                                               ws["counter"].data_ptr())


def _argmax_edge_rows(onehot):
    """A copy of the one-hot rows `onehot` [B, A] whose first rows are the edges of
    torch.argmax: a tie of columns A // 2 and A - 1, a tie across the whole row, and a row of
    NaNs.  torch.argmax gives the first maximum, and 0 for the row of NaNs; the heads that read
    a logged action or label must pick the same column."""
    x = onehot.clone()
    B, A = x.shape
    tie = torch.zeros(A)
    tie[[A // 2, A - 1]] = 1.0
    for r, row in enumerate([tie, torch.ones(A), torch.full((A,), NAN)][:B]):
        x[r] = row
    return x
