"""Device-resident replay (SURVEY.md 8f rank 1): the add / set_priority / index-draw kernels
(csrc/rb200_replay_dev.cu) against (a) CPython's `random` itself, (b) the host path of this
package and (c) golden vectors from the unmodified reference buffers."""
import random

import numpy as np
import pytest
import torch

from tests import golden_util as G
from tests.builders import _build_replay

pytestmark = pytest.mark.gpu


def _stream(n, S, A, seed, p_term=0.05):
    rng = np.random.RandomState(seed)
    return dict(observation=rng.randn(n, S).astype(np.float32),
                action=rng.randint(0, A, n).astype(np.int64),
                reward=rng.randn(n).astype(np.float32), terminal=rng.rand(n) < p_term,
                priority=rng.uniform(0.1, 10.0, n))


def test_device_mt19937_stream_equals_python_random():
    """> 10^6 stratified random.uniform draws: the device stream (MT19937 state uploaded from
    random.getstate()) reproduces CPython's doubles bit for bit, and hands the state back."""
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.replay_memory.device_replay import DeviceReplay

    B = 4096
    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=1 << 14, batch_size=B)
    rb.add_batch(**_stream(1 << 14, 4, 3, 0, p_term=1.0))  # every slot terminal -> all valid
    random.seed(20260923)
    random.random()  # start mid-block
    dr = DeviceReplay(rb)
    qs = torch.empty(260, B, dtype=torch.float64, device="cuda")
    for i in range(260):
        dr.draw_indices(B, queries_out=qs[i])
    got = qs.cpu().numpy()
    dr.raise_if_failed()
    bounds = np.linspace(0.0, 1.0, B + 1)
    want = np.empty_like(got)
    for i in range(260):
        for j in range(B):
            want[i, j] = random.uniform(bounds[j], bounds[j + 1])
    assert got.size > 10 ** 6 and np.array_equal(got, want)
    dr.sync_to_host()  # the host stream continues where the device stopped
    assert random.getstate()[1] is not None
    nxt_dev = random.random()
    random.seed(20260923)
    random.random()
    for _ in range(260 * B):
        random.random()
    assert nxt_dev == random.random()


@pytest.mark.parametrize("name", ["replay_per_h1", "replay_per_h3_wrap_zero", "replay_per_big"])
def test_device_add_and_draw_match_reference(name):
    """Transitions inserted by the device add kernel, indices drawn by the device kernel: the
    validity bitmap and every sampled batch equal the reference's golden vectors."""
    from reagent_b200.replay_memory.device_replay import DeviceReplay

    arrays, meta = G.load(name)
    keys = meta["keys"]
    st = {k: arrays[f"stream.{k}"] for k in keys}
    n0 = 3  # a few host-side adds first (buffer initialisation), the rest on the device
    head = dict(meta, n_add=n0)
    rb = _build_replay({f"stream.{k}": v[:n0] for k, v in st.items()}, head)
    dr = DeviceReplay(rb, stage_rows=64)
    dr.add_rows(**{k: v[n0:] for k, v in st.items()})
    dr.raise_if_failed()
    assert np.array_equal(rb._valid_dev.cpu().numpy().astype(bool), arrays["valid"])
    random.seed(meta["seed"] + 100)
    dr.upload_host_rng()
    for s_i in range(meta["n_samples"]):
        idx = dr.draw_indices(meta["B"])
        batch = rb.sample_transition_batch(batch_size=meta["B"], indices=idx)
        assert np.array_equal(idx.cpu().numpy(), arrays[f"sample{s_i}.indices"].reshape(-1)), s_i
        term = arrays[f"sample{s_i}.terminal"].reshape(-1)
        for f in ("state", "action", "terminal", "step"):
            assert np.array_equal(getattr(batch, f).cpu().numpy(), arrays[f"sample{s_i}.{f}"]), f
        assert np.array_equal(batch.next_state.cpu().numpy()[~term], arrays[f"sample{s_i}.next_state"][~term])
    # back to the host API: identical state to a buffer built entirely on the host
    dr.sync_to_host()
    host = _build_replay(arrays, meta)
    host._flush()  # staged host rows -> device storage
    assert int(rb.add_count) == int(host.add_count) and rb.size == host.size
    assert np.array_equal(rb._is_index_valid.numpy(), host._is_index_valid.numpy())
    assert np.array_equal(rb.sum_tree.heap, host.sum_tree.heap)
    assert rb.sum_tree.max_recorded_priority == host.sum_tree.max_recorded_priority
    assert rb._bad == host._bad
    for k in ("observation", "action", "reward", "terminal"):
        assert torch.equal(rb._store[k], host._store[k]), k


def test_device_set_priority_equals_sequential_host_sets():
    """2^20-leaf tree, 5000 updates with repeated indices, applied in order: the device heap
    equals the host heap (sequential fp64 delta propagation, sum_tree.py:164-189) bit for bit."""
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.replay_memory.device_replay import DeviceReplay

    cap = 1 << 20
    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=cap, batch_size=32)
    rb.add_batch(**_stream(cap, 2, 3, 1))
    dr = DeviceReplay(rb)
    rng = np.random.RandomState(5)
    idx = rng.randint(0, cap, 5000).astype(np.int32)
    idx[::7] = idx[0]  # repeated leaves: order matters
    val = rng.uniform(0.0, 50.0, 5000)
    host_heap = rb.sum_tree.heap.copy()
    from reagent_b200 import _lib

    mx = np.array([rb.sum_tree.max_recorded_priority])
    idx64 = np.ascontiguousarray(idx, dtype=np.int64)  # kept alive across the C call
    _lib.lib().rb200_sumtree_set_host(host_heap.ctypes.data, rb.sum_tree.depth,
                                      idx64.ctypes.data, val.ctypes.data, len(idx),
                                      mx.ctypes.data)
    dr.set_priority(idx, val)
    dr.raise_if_failed()
    assert np.array_equal(dr.tree.cpu().numpy(), host_heap)
    assert float(dr.max_priority.item()) == float(mx[0])
    with pytest.raises(ValueError):
        dr.set_priority(np.array([3], dtype=np.int32), np.array([-1.0]))
        dr.raise_if_failed()


def test_device_retry_exhaustion_raises():
    """prioritized_replay_buffer_test.py:133-145 on the device path."""
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.replay_memory.device_replay import DeviceReplay

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=64, batch_size=8)
    for i in range(40):
        rb.add(observation=np.full(4, i, dtype=np.float32), action=0, reward=float(i),
               terminal=False, priority=1.0)
    rb.set_priority(np.arange(39, dtype=np.int32), np.zeros(39))  # only the invalid slot has mass
    rb._max_sample_attempts = 50
    random.seed(0)
    dr = DeviceReplay(rb)
    dr.draw_indices(8)
    with pytest.raises(RuntimeError, match="Max sample attempts"):
        dr.raise_if_failed()


def test_online_fused_step_equals_host_loop():
    """FusedDqnStep(rng='device', online=True): add one transition + draw + train per step, one
    graph replay each -- same indices and same losses as the host-side loop
    (rb.add -> sample_discrete_dqn_batch with Python's random -> trainer.train_batch)."""
    import bench
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = dict(bench.CONFIGS[2], cap=4096, B=256)
    S, A, B = cfg["S"], cfg["A"], cfg["B"]
    base = _stream(3000, S, A, 3)
    extra = _stream(40, S, A, 4)

    def make():
        rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=cfg["cap"], batch_size=B)
        rb.add_batch(**base)
        return rb, bench.build_trainer(cfg, torch.device("cuda"), seed=3)

    # host loop (no prefetch: add, then draw, then train)
    rb_h, t_h = make()
    random.seed(77)
    losses_h, idx_h = [], []
    for i in range(12):
        rb_h.add(**{k: (v[i].item() if np.ndim(v[i]) == 0 else v[i]) for k, v in extra.items()})
        batch = rb_h.sample_discrete_dqn_batch(B, A)
        idx_h.append(batch.indices.cpu().numpy().reshape(-1).copy())
        losses_h.append(float(t_h.train_batch(batch)))
    # fused online loop
    rb_d, t_d = make()
    random.seed(77)
    fused = FusedDqnStep(t_d, rb_d, B, rng="device", online=True, prefetch=False)
    # (the constructor's warm-up consumed one draw and trained once: redo from a clean state)
    rb_d2, t_d2 = make()
    random.seed(77)
    from reagent_b200.replay_memory.device_replay import DeviceReplay

    dr = DeviceReplay(rb_d2)
    losses_d, idx_d = [], []
    for i in range(12):
        dr.add(**{k: v[i] for k, v in extra.items()})
        idx = dr.draw_indices(B)
        batch = rb_d2.sample_discrete_dqn_batch(B, A, indices=idx)
        idx_d.append(idx.cpu().numpy().copy())
        losses_d.append(float(t_d2.train_batch(batch)))
    for a, b in zip(idx_h, idx_d):
        assert np.array_equal(a, b)
    assert losses_h == losses_d
    # and the captured online step runs, keeps adding, and reports finite losses
    for i in range(12, 30):
        lh = fused.step({k: v[i] for k, v in extra.items()})
    torch.cuda.synchronize()
    assert np.isfinite(float(lh[0]))
    fused.dr.sync_to_host()
    assert int(rb_d.add_count) == 3000 + 18
