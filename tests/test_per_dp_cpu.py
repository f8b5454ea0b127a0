"""Data-parallel prioritized replay without a GPU: FusedDqnStep / FusedPolicyStep argument checks
of per with shard, the trainers that stay single-GPU, and the C ABI checks of the priority
exchange and the PER-semantics tree update."""
import ctypes as C

import numpy as np
import pytest
import torch


def _prioritized_buffer(B=8):
    from reagent_b200.replay_memory import PrioritizedReplayBuffer

    return PrioritizedReplayBuffer(stack_size=1, replay_capacity=64, batch_size=B)


def _dqn():
    import bench

    return bench.build_trainer(dict(bench.CONFIGS[2], S=6, A=3, B=8, sizes=[8, 8]),
                               torch.device("cpu"))


def _sac():
    import bench

    return bench.build_trainer(dict(bench.CONFIGS[4], S=6, A=2, B=8, sizes=[8, 8]),
                               torch.device("cpu"))


@pytest.mark.parametrize("shard", [(0, 2), (1, 4), (0, 3)])
def test_fused_step_per_shard_needs_a_process_group(shard):
    """Past the trainer and buffer checks, per with a sharded world > 1 needs the group whose
    ranks hold the other rows (and world | batch: 8 rows do not split over 3)."""
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep, FusedPolicyStep

    with pytest.raises(ValueError, match="process_group|divisible"):
        FusedDqnStep(_dqn(), _prioritized_buffer(), 8, rng="device", online=True,
                     per=PrioritizedUpdate(), shard=shard)
    with pytest.raises(ValueError, match="process_group|divisible"):
        FusedPolicyStep(_sac(), _prioritized_buffer(), 8, -np.ones(2), np.ones(2),
                        per=PrioritizedUpdate(), shard=shard)


def test_fused_step_per_shard_must_match_the_group():
    """shard = (rank, world) must be the process group's own."""
    import torch.distributed as dist

    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        for shard in [(0, 2), (1, 1)]:
            with pytest.raises(ValueError, match="process group"):
                FusedDqnStep(_dqn(), _prioritized_buffer(), 8, rng="device", online=True,
                             per=PrioritizedUpdate(), shard=shard,
                             process_group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()


def test_device_rng_on_a_uniform_buffer_is_refused_before_touching_it():
    from reagent_b200.replay_memory import ReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep

    rb = ReplayBuffer(stack_size=1, replay_capacity=16, batch_size=4)
    with pytest.raises(NotImplementedError, match="prioritized"):
        FusedDqnStep(_dqn(), rb, 8, rng="device", shard=(0, 2))


class _Buffer:
    """Enough of a buffer for FusedDqnStep's argument checks, which run first."""


@pytest.mark.parametrize("kw", [dict(shard=(0, 2)), dict(process_group=object()),
                                dict(shard=(0, 2), process_group=object(), rng="device")])
def test_parametric_dqn_and_crr_stay_single_gpu(kw):
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import (FullyConnectedActor, FullyConnectedCritic,
                                     FullyConnectedDQN)
    from reagent_b200.training import DiscreteCRRTrainer, ParametricDQNTrainer
    from reagent_b200.training.fused_step import FusedDqnStep

    q = FullyConnectedCritic(4, 3, [8], ["relu"])
    pdqn = ParametricDQNTrainer(q, q.get_target_network())
    actor, q1 = FullyConnectedActor(5, 3, [8], ["relu"]), FullyConnectedDQN(5, 3, [8], ["relu"])
    crr = DiscreteCRRTrainer(actor_network=actor, q1_network=q1, reward_network=None,
                             actor_network_target=actor.get_target_network(),
                             q1_network_target=q1.get_target_network(), actions=["a", "b", "c"],
                             evaluation=EvaluationParameters(calc_cpe_in_training=False))
    for t in (pdqn, crr):
        with pytest.raises(NotImplementedError, match="single-GPU"):
            FusedDqnStep(t, _Buffer(), 8, **kw)


def _exchange_args(**kw):
    from reagent_b200 import _lib

    x = 16  # never dereferenced: the checks reject the call first
    a = _lib.PerExchangeArgsT()
    a.td_target = a.q_selected = a.out = x
    a.alpha, a.eps = 0.6, 1e-6
    a.n_local, a.row0, a.B_global, a.world, a.rank = 4, 4, 8, 2, 1
    a.recv = a.flags = a.epoch = x
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,what", [
    (dict(out=None), b"out"),
    (dict(td_target=None), b"td_target"),
    (dict(q_selected=None), b"q_selected"),
    (dict(recv=None), b"recv"),
    (dict(flags=None), b"flags"),
    (dict(epoch=None), b"epoch"),
    (dict(world=0, rank=0), b"world"),
    (dict(world=257), b"world"),
    (dict(rank=2), b"rank"),
    (dict(rank=-1), b"rank"),
    (dict(n_local=0), b"B_global"),
    (dict(row0=-1), b"B_global"),
    (dict(row0=5), b"B_global"),
    (dict(B_global=7), b"B_global"),
    (dict(row_loss=16, divisor=0.0), b"divisor"),
    (dict(row_loss=16, divisor=float("inf")), b"divisor"),
])
def test_priority_exchange_c_abi_checks(kw, what):
    from reagent_b200 import _lib

    lib = _lib.lib()
    assert lib.rb200_per_priority_exchange(_exchange_args(**kw), None) == -1
    err = lib.rb200_last_error()
    assert b"rb200_per_priority_exchange" in err and what in err
    assert lib.rb200_per_priority_exchange(None, None) == -1


def test_priority_apply_c_abi_checks():
    from reagent_b200 import _lib

    lib = _lib.lib()
    x = C.c_void_p(16)
    args = [x, 3, x, x, 4, x, x, None]
    for i, name in [(0, b"tree"), (2, b"idx"), (3, b"val"), (6, b"status")]:
        bad = list(args)
        bad[i] = None
        assert lib.rb200_per_priority_apply(*bad) == -1
        assert name in lib.rb200_last_error()
    for depth, n in [(-1, 4), (32, 4), (3, 0), (3, -2)]:
        assert lib.rb200_per_priority_apply(x, depth, x, x, n, x, x, None) == -1
        assert b"rb200_per_priority_apply" in lib.rb200_last_error()
