"""Which shapes the wgmma TD kernel (dqn_td_tc_kernel, csrc/rb200_dqn_tc.cu) takes, and how
large its weight-image pack is: rb200_dqn_tc_workspace_bytes against the restatement of
make_plan's admission rules and shared-memory sum in tests/kernel_util._k2_tc_bytes.  A shape
the kernel refuses runs on dqn_td_rows_kernel instead, so an edge that moves silently moves
work between the two kernels; the pinned pairs below name the edges the GPU tests
(test_dqn_td_edges_gpu.py) sit on.  Needs no GPU: the library only plans here."""
import itertools

import pytest

from reagent_b200 import _lib
from tests.kernel_util import _k2_tc_bytes


def _lib_bytes(dims, double_q, do_backward):
    L = len(dims) - 1
    d = _lib.MlpT()
    d.n_layers = L
    off = 0
    for i, v in enumerate(dims):
        d.dims[i] = v
    for l in range(L):
        d.act[l] = _lib.ACT["relu"]
        d.w_off[l] = off
        off += dims[l] * dims[l + 1]
        d.b_off[l] = off
        off += dims[l + 1]
    d.n_params = off
    d.params = 256  # never dereferenced: the call only plans
    return int(_lib.lib().rb200_dqn_tc_workspace_bytes(d, double_q, do_backward))


# (inside, outside): one step past each edge of the shared-memory budget
EDGES = {
    "hidden_width": ([8, 472, 8], [8, 473, 8]),
    "actions": ([8, 8, 141], [8, 8, 142]),
    "state_config2": ([192, 256, 128, 16], [193, 256, 128, 16]),
    "state": ([480, 8, 4], [481, 8, 4]),
}


@pytest.mark.parametrize("edge", sorted(EDGES))
def test_wgmma_plan_edges_sit_where_the_gpu_tests_expect(edge):
    inside, outside = EDGES[edge]
    for dq, bw in itertools.product((0, 1), (0, 1)):
        got_in, got_out = _lib_bytes(inside, dq, bw), _lib_bytes(outside, dq, bw)
        assert got_in == _k2_tc_bytes(inside, dq, bw) > 0, (edge, "inside", inside, dq, bw, got_in)
        assert got_out == _k2_tc_bytes(outside, dq, bw) == 0, (edge, "outside", outside, dq, bw, got_out)


def test_wgmma_plan_matches_the_mirror_over_a_shape_grid():
    S_ = [1, 3, 4, 8, 9, 33, 128, 129, 132, 192, 193, 256, 480, 481, 1000, 32000, 32001]
    H_ = [1, 8, 9, 64, 65, 128, 129, 256, 300, 384, 385, 472, 473, 512, 513]
    A_ = [1, 2, 9, 16, 128, 129, 141, 142, 256, 257]
    shapes = []
    for S, H, A in itertools.product(S_, H_, A_):
        shapes += [[S, A], [S, H, A], [S, H, 16, A], [S] + [H] * 3 + [A]]
    for L in range(1, 10):
        for H in (8, 16, 65, 129, 300):
            shapes.append([33] + [H] * (L - 1) + [9])
            shapes.append([129] + [H] * (L - 1) + [141])
    n_in = n_out = 0
    for dims in shapes:
        for dq, bw in itertools.product((0, 1), (0, 1)):
            want = _k2_tc_bytes(dims, dq, bw)
            if len(dims) - 1 > _lib.MAX_LAYERS:
                assert want == 0
                continue
            assert _lib_bytes(dims, dq, bw) == want, (dims, dq, bw, want)
            n_in += want > 0
            n_out += want == 0
    # the grid straddles the budget: both sides well populated
    assert n_in > 1000 and n_out > 1000, (n_in, n_out)


def test_forward_only_pack_has_no_backward_images():
    dims = [33, 300, 129, 9]
    fwd_only, with_bwd = _lib_bytes(dims, 1, 0), _lib_bytes(dims, 1, 1)
    assert 0 < fwd_only < with_bwd
    assert with_bwd == _k2_tc_bytes(dims, 1, 1) and fwd_only == _k2_tc_bytes(dims, 1, 0)
