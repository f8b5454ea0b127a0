"""Prioritized replay for SACTrainer and TD3Trainer without a GPU: the weighted oracles against
the reference's SAC and TD3 goldens, the twin-critic priorities, and the argument checks of
FusedPolicyStep and of `importance_weights`."""

import numpy as np
import pytest
import torch

from oracle import per_ac_oracle as PA
from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import SAC_CASES, TD3_CASES
from tests.golden_util import _cmp_losses, _cmp_net


@pytest.mark.parametrize("name", SAC_CASES)
def test_weighted_sac_oracle_with_unit_weights_reproduces_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    actor = G.oracle_net(arrays, "actor0", acts)
    q1 = G.oracle_net(arrays, "q1_0", acts)
    q2 = G.oracle_net(arrays, "q2_0", acts) if meta["twin"] else None
    st = O.SacState(actor, q1, q2, lr=meta["lr"], entropy_temperature=meta["entropy_temperature"],
                    learn_alpha=meta["learn_alpha"], target_entropy=meta["target_entropy"])
    batch = G.batch_tensors(arrays)
    w = torch.ones(batch["reward"].shape[0])
    for it in range(meta["n_updates"]):
        out = PA.weighted_sac_update(st, batch, torch.from_numpy(arrays[f"noise{it}.next"]),
                                     torch.from_numpy(arrays[f"noise{it}.cur"]), w,
                                     gamma=meta["gamma"], tau=meta["tau"],
                                     backprop_through_log_prob=meta["backprop"])
        _cmp_losses(out["losses"], arrays["losses"][it], 2e-6)
        if it == 0:
            names = ["q1"] + (["q2"] if meta["twin"] else []) + ["actor"] + (
                ["alpha"] if meta["learn_alpha"] else [])
            for oi, nm in enumerate(names):
                for pi, g in enumerate(out["grads"][nm]):
                    assert G.rel_err(g, arrays[f"grad0.opt{oi}.{pi}"]) < 2e-5, (nm, pi)
    _cmp_net(st.actor, arrays, "actorN", 1e-5)
    _cmp_net(st.q1, arrays, "q1_N", 1e-5)
    _cmp_net(st.q1t, arrays, "q1t_N", 1e-5)
    if meta["twin"]:
        _cmp_net(st.q2, arrays, "q2_N", 1e-5)
        _cmp_net(st.q2t, arrays, "q2t_N", 1e-5)
    if meta["learn_alpha"]:
        assert G.rel_err(st.log_alpha, arrays["log_alpha_N"]) < 1e-6


@pytest.mark.parametrize("name", TD3_CASES)
def test_weighted_td3_oracle_with_unit_weights_reproduces_reference(name):
    arrays, meta = G.load(name)
    actor = G.oracle_net(arrays, "actor0", meta["acts"] + ["tanh"])
    cacts = meta["acts"] + ["linear"]
    q1 = G.oracle_net(arrays, "q1_0", cacts)
    q2 = G.oracle_net(arrays, "q2_0", cacts) if meta["twin"] else None
    st = O.Td3State(actor, q1, q2, lr=meta["lr"])
    batch = G.batch_tensors(arrays)
    w = torch.ones(batch["reward"].shape[0])
    for it in range(meta["n_updates"]):
        out = PA.weighted_td3_update(st, batch, torch.from_numpy(arrays[f"noise{it}.next"]), it, w,
                                     gamma=meta["gamma"], tau=meta["tau"],
                                     noise_variance=meta["noise_variance"],
                                     noise_clip=meta["noise_clip"],
                                     delayed_policy_update=meta["delay"])
        _cmp_losses(out["losses"], arrays["losses"][it], 2e-6)
    _cmp_net(st.actor, arrays, "actorN", 1e-5)
    _cmp_net(st.actor_t, arrays, "actort_N", 1e-5)
    _cmp_net(st.q1, arrays, "q1_N", 1e-5)
    _cmp_net(st.q1t, arrays, "q1t_N", 1e-5)
    if meta["twin"]:
        _cmp_net(st.q2, arrays, "q2_N", 1e-5)
        _cmp_net(st.q2t, arrays, "q2t_N", 1e-5)


def test_weighted_critic_loss_scales_rows_and_leaves_the_actor_alone():
    """Doubling every weight doubles both critic losses and gradients, the actor's gradient
    does not depend on the weights, and the TD error is the larger critic's |q - y|."""
    gen = torch.Generator().manual_seed(0)
    S, A, B = 5, 2, 6

    def run(w):
        g2 = torch.Generator().manual_seed(1)
        actor = O.make_net([S, 8, A], ["relu", "tanh"], g2)
        q1 = O.make_net([S + A, 8, 1], ["relu", "linear"], g2)
        q2 = O.make_net([S + A, 8, 1], ["relu", "linear"], g2)
        st = O.Td3State(actor, q1, q2, lr=1e-3)
        return PA.weighted_td3_update(st, batch, noise, 0, w, gamma=0.9, tau=0.1)

    batch = {"state": torch.randn(B, S, generator=gen), "next_state": torch.randn(B, S, generator=gen),
             "action": torch.rand(B, A, generator=gen) * 2 - 1, "reward": torch.randn(B, 1, generator=gen),
             "not_terminal": torch.ones(B, 1)}
    noise = torch.randn(B, A, generator=gen)
    w = torch.rand(B, generator=gen) + 0.1
    a, b = run(w), run(2 * w)
    for i in range(2):
        assert abs(b["losses"][i] - 2 * a["losses"][i]) <= 1e-6 * abs(b["losses"][i])
    for ga, gb in zip(a["grads"]["q1"], b["grads"]["q1"]):
        assert torch.allclose(gb, 2 * ga, rtol=1e-5, atol=1e-7)
    for ga, gb in zip(a["grads"]["actor"], b["grads"]["actor"]):
        assert torch.equal(ga, gb)
    assert torch.equal(a["td_error"], b["td_error"])
    want = torch.maximum((a["q1_value"] - a["target"].reshape(-1)).abs(),
                         (a["q2_value"] - a["target"].reshape(-1)).abs())
    assert torch.equal(a["td_error"], want)


def test_twin_td_priorities_known_values():
    p = PA.twin_td_priorities([1.0, 0.0], [0.5, -3.0], [0.0, 1.0], 0.5, 0.0)
    assert p.dtype == np.float64 and np.array_equal(p, np.sqrt([1.0, 4.0]))
    p = PA.twin_td_priorities([2.0], None, [0.5], 1.0, 1e-6)
    assert p[0] == 1.5 + 1e-6
    assert np.isnan(PA.twin_td_priorities([np.nan], [0.0], [0.0], 0.6, 1e-6)[0])


def _cpu_trainers(delay=2):
    import bench
    from reagent_b200.training import TD3Trainer

    sac = bench.build_trainer(dict(bench.CONFIGS[4], S=6, A=2, B=8, sizes=[8, 8]), torch.device("cpu"))
    td3 = bench.build_trainer(dict(bench.CONFIGS[5], S=6, A=2, B=8, sizes=[8, 8]), torch.device("cpu"))
    assert type(td3) is TD3Trainer and td3.delayed_policy_update == delay
    return sac, td3


class _Fake:
    """Just enough of a buffer for FusedPolicyStep's argument checks, which run first."""


@pytest.mark.parametrize("kw,exc", [
    (dict(rng="host"), ValueError),
    (dict(prefetch=True), ValueError),
    (dict(shard=(0, 2)), NotImplementedError),
    (dict(process_group=object()), NotImplementedError),
    (dict(slots=0), ValueError),
])
@pytest.mark.parametrize("with_per", [False, True])
@pytest.mark.parametrize("which", [0, 1])
def test_fused_policy_step_argument_errors(kw, exc, with_per, which):
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedPolicyStep

    trainer = _cpu_trainers()[which]
    per = PrioritizedUpdate() if with_per else None
    with pytest.raises(exc):
        FusedPolicyStep(trainer, _Fake(), 8, -np.ones(2), np.ones(2), per=per, **kw)


def test_fused_policy_step_needs_a_prioritized_buffer():
    from reagent_b200.replay_memory import ReplayBuffer
    from reagent_b200.training.fused_step import FusedPolicyStep

    sac, _ = _cpu_trainers()
    rb = ReplayBuffer(stack_size=1, replay_capacity=16, batch_size=4)
    with pytest.raises(NotImplementedError, match="prioritized"):
        FusedPolicyStep(sac, rb, 4, -np.ones(2), np.ones(2))


def test_fused_policy_step_rejects_other_trainer_types():
    """Only the exact types SACTrainer and TD3Trainer: a subclass could change what the
    workspace's TD errors mean.  Discrete trainers take FusedDqnStep."""
    import bench
    from reagent_b200.training import SACTrainer
    from reagent_b200.training.fused_step import FusedPolicyStep

    sac, _ = _cpu_trainers()

    class MySAC(SACTrainer):
        pass

    sac.__class__ = MySAC
    dqn = bench.build_trainer(dict(bench.CONFIGS[2], S=6, A=3, B=8, sizes=[8, 8]), torch.device("cpu"))
    for t in (_Fake(), sac, dqn):
        with pytest.raises(NotImplementedError, match="SACTrainer and TD3Trainer"):
            FusedPolicyStep(t, _Fake(), 8, -np.ones(2), np.ones(2))


def _cpu_batch(B=8, S=6, A=2):
    from reagent_b200.core import types as rlt

    return rlt.PolicyNetworkInput(
        state=rlt.FeatureData(torch.randn(B, S)), next_state=rlt.FeatureData(torch.randn(B, S)),
        action=rlt.FeatureData(torch.zeros(B, A)), next_action=rlt.FeatureData(torch.zeros(B, A)),
        reward=torch.zeros(B, 1), not_terminal=torch.ones(B, 1), step=None, time_diff=None,
        extras=rlt.ExtraData())


@pytest.mark.parametrize("which", [0, 1])
def test_importance_weights_are_validated_before_any_launch(which):
    """A wrong dtype or shape raises ValueError (DQNTrainer's message) before the CUDA checks."""
    trainer = _cpu_trainers()[which]
    batch = _cpu_batch()
    for bad in (torch.ones(8, dtype=torch.float64), torch.ones(9), torch.ones(8, 1),
                torch.ones(8, dtype=torch.float16)):
        with pytest.raises(ValueError, match="importance_weights"):
            trainer.train_batch(batch, 0, importance_weights=bad)
    assert trainer.all_batches_processed == 0
