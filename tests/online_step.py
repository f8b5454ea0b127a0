"""The checks every captured online step shares (FusedDqnStep(rng="device", online=True) and
FusedPolicyStep): synthetic transitions, n online steps run captured or eagerly, captured
against eager bit for bit, the online loop against a host replica of the reference buffer, a
NaN reward, and the sum-tree helpers of the prioritized-replay tests.

`online_steps` is the only test code that runs the step's eager twin through its internals
(`_one_update`, `dr.stage`, `dr.launch_add`), so a change to them is made here once."""
import random

import numpy as np
import pytest
import torch


def transition_stream(n, seed, S=None, A=None, cfg=None):
    """n synthetic transitions: discrete actions in [0, A) on S-wide states with 5 % terminals,
    or, given a bench config, bench.synth_stream's (continuous actions for SAC / TD3)."""
    if cfg is not None:
        import bench

        return bench.synth_stream(n, seed, cfg)
    rng = np.random.RandomState(seed)
    return dict(observation=rng.randn(n, S).astype(np.float32),
                action=rng.randint(0, A, n).astype(np.int64),
                reward=rng.randn(n).astype(np.float32), terminal=rng.rand(n) < 0.05,
                priority=rng.uniform(0.1, 10.0, n))


def prioritized_buffer(cfg, base):
    """A PrioritizedReplayBuffer of cfg["cap"] rows holding the transitions `base`."""
    from reagent_b200.replay_memory import PrioritizedReplayBuffer

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=cfg["cap"], batch_size=cfg["B"])
    rb.add_batch(**base)
    return rb


def bench_setup(cfg, base, seed=3):
    """prioritized_buffer(cfg, base) and bench's trainer for cfg."""
    import bench

    rb = prioritized_buffer(cfg, base)
    return rb, bench.build_trainer(cfg, torch.device("cuda"), seed=seed)


def host_add(rb, tr):
    """ReplayBuffer.add of one transition whose values are numpy scalars or rows."""
    rb.add(**{k: (v.item() if np.ndim(v) == 0 and hasattr(v, "item") else v)
              for k, v in tr.items()})


def drawn_indices(fused):
    """The replay indices the step's last update drew, on the host."""
    return fused._idx_buf[0].cpu().numpy().copy()


def online_steps(fused, extra, n, captured, drop_priority=None, scalar_loss=True,
                 before_step=None):
    """Yields the loss of each of n online steps adding extra[i], through graph replay or through
    eager launches of the same stage, add and update.  `drop_priority(i)`: transition i has no
    priority (the step gives it the max priority under per).  The loss is float(loss[0]), or a
    host copy of the whole loss tensor.  `before_step()` runs before each step."""
    from_max = fused.per is not None
    for i in range(n):
        if before_step is not None:
            before_step()
        tr = {k: v[i] for k, v in extra.items()}
        if drop_priority is not None and drop_priority(i):
            del tr["priority"]
        if captured:
            out = fused.step(tr)
            torch.cuda.current_stream().synchronize()
            yield float(out[0]) if scalar_loss else out.clone()
        else:
            fused.dr.stage(0, 0, priority_from_max=from_max, **tr)
            fused.dr.launch_add(1, slot=0, priority_from_max=from_max)
            out = fused._one_update(None)
            yield float(out) if scalar_loss else out.cpu()
    torch.cuda.synchronize()
    fused.dr.raise_if_failed()


def params(*modules):
    return [p.detach().clone() for m in modules for p in m.parameters()]


def tree(fused):
    """The device sum tree and its max priority."""
    return [fused.dr.tree.clone(), float(fused.dr.max_priority)]


def _bits(t):
    t = t.detach().contiguous()
    if not t.is_floating_point():
        return t
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def same_bits(a, b):
    """Tensors equal bit for bit (-0.0 is not 0.0), nested lists item by item, the rest by ==."""
    if isinstance(a, torch.Tensor):
        return (isinstance(b, torch.Tensor) and a.shape == b.shape and a.dtype == b.dtype
                and torch.equal(_bits(a), _bits(b)))
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same_bits(x, y) for x, y in zip(a, b))
    return a == b


def assert_captured_equals_eager(setup, extra, n, snapshot, drop_priority=None,
                                 scalar_loss=True):
    """Runs `setup() -> (fused, before_step or None)` twice from the same seeds, n online steps
    captured and then eagerly: the losses (all finite) and `snapshot(fused)` agree bit for bit.
    Returns the captured run's snapshot."""
    runs = []
    for captured in (True, False):
        fused, before_step = setup()
        losses = list(online_steps(fused, extra, n, captured, drop_priority, scalar_loss,
                                   before_step))
        runs.append((losses, snapshot(fused)))
    (l0, s0), (l1, s1) = runs
    assert same_bits(l0, l1)
    assert all(bool(torch.isfinite(torch.as_tensor(x)).all()) for x in l0)
    assert same_bits(s0, s1)
    return s0


def assert_matches_host_replica(make_fused, rb_h, extra, sample, want_priorities=None,
                                steps=30):
    """`make_fused()` builds the prioritized online step from Python's random state at seed 77;
    `rb_h` holds the same transitions.  After the warm-up update and each of `steps` steps (every
    third transition without a priority), the host buffer's `sample(rb_h)` draws the step's
    indices and takes its priorities, which are within 4 fp64 ulp of
    `want_priorities(trainer)` when given.  Ends with the device tree equal to the host's, bit
    for bit.  Returns the step."""
    random.seed(77)
    saved = random.getstate()
    fused = make_fused()
    random.setstate(saved)

    def replica_update():
        torch.cuda.synchronize()
        idx_h = sample(rb_h).indices.cpu().numpy().reshape(-1)
        assert np.array_equal(idx_h, drawn_indices(fused))
        pr = fused.priorities.cpu().numpy()
        if want_priorities is not None:
            assert ulps(pr, want_priorities(fused.trainer)).max() <= 4
        rb_h.set_priority(idx_h.astype(np.int32), pr)

    replica_update()  # the constructor's warm-up update
    for i in range(steps):
        tr = {k: v[i] for k, v in extra.items()}
        if i % 3 == 1:
            del tr["priority"]
        fused.step(tr)
        host_tr = dict(tr)
        host_tr.setdefault("priority", rb_h.sum_tree.max_recorded_priority)
        host_add(rb_h, host_tr)
        replica_update()
    fused.dr.sync_to_host()
    assert np.array_equal(fused.rb.sum_tree.heap, rb_h.sum_tree.heap)
    assert fused.rb.sum_tree.max_recorded_priority == rb_h.sum_tree.max_recorded_priority
    return fused


def assert_nan_reward_raises(fused, extra):
    """A NaN reward, drawn by the next update through its huge priority, raises
    FloatingPointError within the following steps."""
    bad = {k: v[0] for k, v in extra.items()}
    bad["reward"] = np.float32("nan")
    bad["priority"] = 1e9  # drawn by the next update
    with pytest.raises(FloatingPointError):
        fused.step(bad)
        for i in range(1, 10):
            fused.step({k: v[i] for k, v in extra.items()})
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# sum tree
# ---------------------------------------------------------------------------
def filled_heap(cap, rng):
    """(heap, depth, max priority) of a host sum tree with cap leaves uniform in [0, 10)."""
    from reagent_b200 import _lib

    depth = int(np.ceil(np.log2(cap))) if cap > 1 else 0
    heap = np.zeros((1 << (depth + 1)) - 1)
    idx = np.arange(cap, dtype=np.int64)
    val = rng.uniform(0.0, 10.0, cap)
    mx = np.array([1.0])
    assert _lib.lib().rb200_sumtree_set_host(heap.ctypes.data, depth, idx.ctypes.data,
                                             val.ctypes.data, cap, mx.ctypes.data) == 0
    return heap, depth, mx


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def rows_update(heap_d, depth, idx, row_loss, D, per, p, dm, st):
    """rb200_per_priority_update_rows: priorities of the per-row losses / D into the tree."""
    from reagent_b200 import _lib

    _lib.check(_lib.lib().rb200_per_priority_update_rows(
        heap_d.data_ptr(), depth, idx.data_ptr(), row_loss.data_ptr(), idx.numel(), float(D),
        per.alpha, per.eps, p.data_ptr(), dm.data_ptr(), st.data_ptr(), _lib.cur_stream()))
    torch.cuda.synchronize()
