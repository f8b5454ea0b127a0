"""wgmma wide Linear forward (rb200_linear_forward -> tc_linear_fwd_kernel) vs an
fp64 torch reference: full tiles, ragged rows / columns / K, scalar-load path, activations."""
import pytest
import torch

from tests import golden_util as G

pytestmark = pytest.mark.gpu


def _run(B, K, N, act):
    from reagent_b200 import _lib

    g = torch.Generator().manual_seed(B * 7 + K * 3 + N)
    x = torch.randn(B, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g) * 0.1
    ref = x.double() @ W.double().t() + b.double()
    if act == "relu":
        ref = torch.relu(ref)
    elif act == "tanh":
        ref = torch.tanh(ref)
    xd, Wd, bd = x.cuda(), W.cuda().contiguous(), b.cuda()
    out = torch.empty(B, N, device="cuda")
    rc = _lib.lib().rb200_linear_forward(Wd.data_ptr(), bd.data_ptr(), _lib.ACT[act if act else "linear"],
                                         K, N, xd.data_ptr(), B, out.data_ptr(), _lib.cur_stream())
    _lib.check(rc, "rb200_linear_forward")
    torch.cuda.synchronize()
    return G.rel_err(out, ref.float())


@pytest.mark.parametrize("B,K,N,act", [
    (128, 32, 128, None),        # exactly one tile, one k-chunk
    (128, 128, 256, "relu"),     # 4 chunks (ring wraps), 2 column tiles
    (4096, 128, 6400, None),     # QR-DQN head of BASELINE config 3
    (300, 100, 200, "tanh"),     # ragged rows / cols, K not a multiple of 32
    (256, 36, 130, None),        # K tail quad, 2 columns in the last tile
    (129, 7, 129, "relu"),       # scalar-load path (K % 4 != 0)
    (64, 128, 6400, None),       # batch < 128 -> row-tile mma.sync path
])
def test_linear_forward(B, K, N, act):
    assert _run(B, K, N, act) < 1e-5


@pytest.mark.parametrize("B,K,N,act", [
    (4096, 128, 6400, "relu"),   # QR-DQN head of BASELINE config 3 (13 split-K slices)
    (4096, 128, 1632, "relu"),   # C51 head: 32 actions x 51 atoms (ragged last chunk: 1632 = 51 * 32)
    (300, 100, 1028, "tanh"),    # ragged rows / columns, contraction tail quad
    (256, 260, 1024, None),      # three column tiles, no activation below
])
def test_linear_backward_dx_tc(B, K, N, act):
    """rb200_linear_backward_dx_tc (split-K wgmma) vs fp64 torch and vs the mma.sync kernel it
    replaces for wide heads: out = (dz . W) * act'(h_prev)."""
    from reagent_b200 import _lib

    lib = _lib.lib()
    g = torch.Generator().manual_seed(B + K * 5 + N)
    dz = torch.randn(B, N, generator=g)
    W = torch.randn(N, K, generator=g) / N ** 0.5
    pre = torch.randn(B, K, generator=g)
    h = torch.relu(pre) if act == "relu" else (torch.tanh(pre) if act == "tanh" else pre)
    ref = dz.double() @ W.double()
    if act == "relu":
        ref = ref * (h > 0).double()
    elif act == "tanh":
        ref = ref * (1.0 - h.double() ** 2)
    dzd, Wd, hd = dz.cuda(), W.cuda().contiguous(), h.cuda()
    nbytes = int(lib.rb200_linear_backward_dx_tc_scratch_bytes(K, N, B))
    assert nbytes > 0
    scratch = torch.empty(nbytes // 4, device="cuda")
    out = torch.empty(B, K, device="cuda")
    a = _lib.ACT[act if act else "linear"]
    rc = lib.rb200_linear_backward_dx_tc(Wd.data_ptr(), K, N, dzd.data_ptr(), hd.data_ptr(), a, B,
                                         out.data_ptr(), scratch.data_ptr(), nbytes, _lib.cur_stream())
    _lib.check(rc, "rb200_linear_backward_dx_tc")
    out2 = torch.empty(B, K, device="cuda")
    rc = lib.rb200_linear_backward_dx(Wd.data_ptr(), K, N, dzd.data_ptr(), hd.data_ptr(), a, B,
                                      out2.data_ptr(), _lib.cur_stream())
    _lib.check(rc, "rb200_linear_backward_dx")
    torch.cuda.synchronize()
    assert G.rel_err(out, ref.float()) < 1e-5
    assert G.rel_err(out, out2) < 1e-5
    # deterministic: the slices are added in a fixed order
    out3 = torch.empty(B, K, device="cuda")
    lib.rb200_linear_backward_dx_tc(Wd.data_ptr(), K, N, dzd.data_ptr(), hd.data_ptr(), a, B,
                                    out3.data_ptr(), scratch.data_ptr(), nbytes, _lib.cur_stream())
    torch.cuda.synchronize()
    assert torch.equal(out, out3)


def test_linear_backward_dx_tc_declines_small_shapes():
    from reagent_b200 import _lib

    lib = _lib.lib()
    assert lib.rb200_linear_backward_dx_tc_scratch_bytes(128, 512, 4096) == 0   # narrow head
    assert lib.rb200_linear_backward_dx_tc_scratch_bytes(128, 6400, 64) == 0    # small batch
    assert lib.rb200_linear_backward_dx_tc_scratch_bytes(126, 6400, 4096) == 0  # unaligned rows
