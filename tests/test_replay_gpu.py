"""GPU parity of the fused replay-sample kernel against golden vectors from the unmodified
reference buffers (oracle/make_golden.py::replay_case): bit-exact indices and gathered
fields, fp32-exact n-step rewards, sampling probabilities."""
import random

import numpy as np
import pytest
import torch

from tests import golden_util as G
from tests.builders import _build_replay

pytestmark = pytest.mark.gpu

CASES = ["replay_uniform_h1", "replay_uniform_h3_wrap", "replay_uniform_h5_cont",
         "replay_uniform_stack3", "replay_per_h1", "replay_per_h3_wrap_zero", "replay_per_big"]


def _cmp(name, got, want, terminal=None):
    got = got.cpu().numpy()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    assert got.dtype == want.dtype, (name, got.dtype, want.dtype)
    if name.split(".")[-1].startswith("next_") and terminal is not None:
        # "When the transition is terminal next_state_batch has undefined contents"
        # (circular_replay_buffer.py:621): the reference may read np.empty() memory there.
        keep = ~terminal.reshape(-1)
        got, want = got[keep], want[keep]
    if name.split(".")[-1] in ("reward",):
        # n-step fold: same fp32 products; summation order of torch.sum(dim=1) may differ
        np.testing.assert_allclose(got, want, rtol=2e-6, atol=1e-6, err_msg=name)
    else:
        assert np.array_equal(got, want), name


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("bulk", [False, True])
def test_replay_matches_reference(name, bulk):
    arrays, meta = G.load(name)
    if bulk and meta["stack"] != 1:
        pytest.skip("bulk loader is stack_size == 1 only")
    rb = _build_replay(arrays, meta, bulk)
    assert np.array_equal(rb._is_index_valid.numpy(), arrays["valid"])
    assert rb.size == int(arrays["valid"].sum())
    random.seed(meta["seed"] + 100)
    torch.manual_seed(meta["seed"] + 100)
    np.random.seed(meta["seed"] + 100)
    for s_i in range(meta["n_samples"]):
        batch = rb.sample_transition_batch(batch_size=meta["B"])
        for f in batch._fields:
            key = f"sample{s_i}.{f}"
            if key in arrays:
                _cmp(key, getattr(batch, f), arrays[key], arrays[f"sample{s_i}.terminal"])
    allb = rb.sample_all_valid_transitions()
    for f in allb._fields:
        key = f"all.{f}"
        if key in arrays:
            _cmp(key, getattr(allb, f), arrays[key], arrays["all.terminal"])
    if meta["prioritized"]:
        idx = np.arange(0, min(meta["cap"], 32), dtype=np.int32)
        assert np.array_equal(rb.get_priority(idx), arrays["get_priority"])
        rb.set_priority(idx, arrays["set_priority.values"])
        assert rb.sum_tree._total_priority() == arrays["tree_root_after_set"][0]
        batch = rb.sample_transition_batch(batch_size=meta["B"])
        _cmp("after_set.indices", batch.indices, arrays["after_set.indices"])
        _cmp("after_set.sampling_probabilities", batch.sampling_probabilities,
             arrays["after_set.sampling_probabilities"])


def test_per_retry_path_and_exhaustion():
    """prioritized_replay_buffer_test.py:120-145: zero-priority never sampled; attempts
    exhausted raises RuntimeError."""
    from reagent_b200.replay_memory import PrioritizedReplayBuffer

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=64, batch_size=8)
    for i in range(40):
        rb.add(observation=np.full(4, i, dtype=np.float32), action=0, reward=float(i),
               terminal=False, priority=1.0)
    # index 39 (cursor-1) carries priority but is not yet a valid transition -> retries
    random.seed(0)
    for _ in range(20):
        b = rb.sample_transition_batch(batch_size=32)
        idx = b.indices.cpu().numpy().reshape(-1)
        assert (idx != 39).all() and (idx < 39).all()
    # only the invalid index has mass -> attempts exhausted
    rb.set_priority(np.arange(39, dtype=np.int32), np.zeros(39))
    rb._max_sample_attempts = 50
    with pytest.raises(RuntimeError, match="Max sample attempts"):
        rb.sample_transition_batch(batch_size=8)


def test_fused_normalisation_in_gather():
    """state/next_state normalised on the fly == Preprocessor.forward on the raw gather."""
    from reagent_b200.core.parameters import NormalizationParameters as NP
    from reagent_b200.preprocessing import Preprocessor
    from reagent_b200.replay_memory import ReplayBuffer

    rng = np.random.RandomState(0)
    S, n = 16, 500
    rb = ReplayBuffer(replay_capacity=1024, batch_size=64)
    rb.add_batch(observation=rng.randn(n, S).astype(np.float32) * 4,
                 action=rng.randint(0, 3, n).astype(np.int64),
                 reward=rng.randn(n).astype(np.float32), terminal=rng.rand(n) < 0.05)
    norm = {i: NP("CONTINUOUS", mean=0.1 * i, stddev=1.0 + 0.2 * i) for i in range(S)}
    pre = Preprocessor(norm).eval()
    torch.manual_seed(3)
    raw = rb.sample_transition_batch(batch_size=64)
    rb.set_state_preprocessor(pre)
    torch.manual_seed(3)
    fused = rb.sample_transition_batch(batch_size=64)
    assert torch.equal(raw.indices, fused.indices)
    ones = torch.ones_like(raw.state, dtype=torch.uint8)
    assert torch.equal(pre(raw.state, ones), fused.state)
    assert torch.equal(pre(raw.next_state, ones), fused.next_state)


def test_preprocessor_matches_reference():
    from reagent_b200.core.parameters import NormalizationParameters as NP
    from reagent_b200.preprocessing import Preprocessor

    arrays, meta = G.load("preprocessor_all_types")
    norm = {int(k): NP(**v) for k, v in meta["spec"].items()}
    p = Preprocessor(norm).eval()
    assert list(p.sorted_features) == list(arrays["sorted_features"])
    x = torch.from_numpy(arrays["x"]).cuda()
    pres = torch.from_numpy(arrays["presence"]).cuda()
    out = p(x, pres)
    np.testing.assert_allclose(out.cpu().numpy(), arrays["out"], rtol=2e-6, atol=2e-6)
    out2 = p(x, torch.ones_like(pres))
    np.testing.assert_allclose(out2.cpu().numpy(), arrays["out_all_present"], rtol=2e-6, atol=2e-6)
    # float presence and bool presence behave like uint8
    np.testing.assert_array_equal(p(x, pres.float()).cpu().numpy(), out.cpu().numpy())
    np.testing.assert_array_equal(p(x, pres.bool()).cpu().numpy(), out.cpu().numpy())
    # training mode range check (preprocessor.py:576-599): PROBABILITY stays within range
    p.train()
    p(x, pres)


@pytest.mark.parametrize("name", ["replay_uniform_h3_wrap", "replay_per_h3_wrap_zero"])
def test_checkpoint_load_rebuilds_device_mirrors(name, tmp_path):
    """save() / load() (circular_replay_buffer.py:810-897 of the reference): loading into a
    buffer whose device store, priority mirror and pinned staging block hold OTHER data must
    leave it sampling exactly like the buffer that was saved."""
    arrays, meta = G.load(name)
    src = _build_replay(arrays, meta, bulk=True)
    src.save(str(tmp_path), 3)

    # same add history (validity bookkeeping is private state and, as in the reference, not
    # part of a checkpoint), different contents
    other = {k: np.array(v, copy=True) for k, v in arrays.items()}
    rng = np.random.RandomState(5)
    for k in meta["keys"]:
        v = other[f"stream.{k}"]
        if k == "terminal":
            continue
        if k == "priority":
            other[f"stream.{k}"] = rng.uniform(0.5, 2.0, v.shape)
        elif np.issubdtype(v.dtype, np.floating):
            other[f"stream.{k}"] = rng.standard_normal(v.shape).astype(v.dtype)
    dst = _build_replay(other, meta, bulk=True)
    B = meta["B"]
    random.seed(3); np.random.seed(3); torch.manual_seed(3)
    dst.sample_transition_batch(batch_size=B)  # device mirrors of the OLD contents now exist
    dst.load(str(tmp_path), 3)
    assert dst._stage_n == 0

    for rb in (src, dst):
        random.seed(11); np.random.seed(11); torch.manual_seed(11)
        rb._out = rb.sample_transition_batch(batch_size=B)
    for f in src._out._fields:
        a, b = getattr(src._out, f), getattr(dst._out, f)
        assert torch.equal(torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()), f
