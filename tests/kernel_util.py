"""Constants and launch helpers of the kernel-level tests (the layer, Adam and loss-reduction
kernels) that more than one test module uses."""
import ctypes as C

import numpy as np
import torch

from reagent_b200 import _lib

NAN = float("nan")
NUM_SMS = 132


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
