"""Pins the SAC value-network / CRR restatement (oracle/sac_value_oracle.py) against golden
vectors of the UNMODIFIED reference SACTrainer (oracle/make_sac_value_golden.py), and checks
the trainer's, builder's and manager's construction on the CPU."""
import pytest
import torch

from oracle import sac_value_oracle as V
from tests import golden_util as G
from tests.golden_cases import SAC_VALUE_CASES, opt_names


def oracle_state(arrays, meta):
    acts = meta["acts"] + ["linear"]
    actor = G.oracle_net(arrays, "actor0", acts)
    q1 = G.oracle_net(arrays, "q1_0", acts)
    q2 = G.oracle_net(arrays, "q2_0", acts) if meta["twin"] else None
    value = G.oracle_net(arrays, "v0", acts)
    return V.SacValueState(actor, q1, q2, value, lr=meta["lr"],
                           entropy_temperature=meta["entropy_temperature"],
                           learn_alpha=meta["learn_alpha"], target_entropy=meta["target_entropy"],
                           logged_action_uniform_prior=meta["uniform_prior"], crr=meta["crr"])


def _cmp_net(net, arrays, prefix, tol):
    for i in range(len(net["W"])):
        assert G.rel_err(net["W"][i], arrays[f"{prefix}.W{i}"]) < tol, f"{prefix}.W{i}"
        assert G.rel_err(net["b"][i], arrays[f"{prefix}.b{i}"]) < tol, f"{prefix}.b{i}"


@pytest.mark.parametrize("name", SAC_VALUE_CASES)
def test_sac_value_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    st = oracle_state(arrays, meta)
    batch = G.batch_tensors(arrays)
    names = opt_names(meta)
    for it in range(meta["n_updates"]):
        out = V.sac_value_update(st, batch, torch.from_numpy(arrays[f"noise{it}.cur"]),
                                 gamma=meta["gamma"], tau=meta["tau"])
        ref = arrays["losses"][it]
        assert len(out["losses"]) == len(ref) == len(names)
        for g, w in zip(out["losses"], ref):
            assert abs(g - w) <= 2e-6 * max(1.0, abs(w)), (it, out["losses"], ref)
        if it == 0:
            for oi, nm in enumerate(names):
                for pi, g in enumerate(out["grads"][nm]):
                    assert G.rel_err(g, arrays[f"grad0.opt{oi}.{pi}"]) < 2e-5, (nm, pi)
    _cmp_net(st.actor, arrays, "actorN", 1e-5)
    _cmp_net(st.q1, arrays, "q1_N", 1e-5)
    if meta["twin"]:
        _cmp_net(st.q2, arrays, "q2_N", 1e-5)
    _cmp_net(st.value, arrays, "vN", 1e-5)
    _cmp_net(st.value_t, arrays, "vt_N", 1e-5)
    if meta["learn_alpha"]:
        assert G.rel_err(st.log_alpha, arrays["log_alpha_N"]) < 1e-5


def test_crr_weight_fn_matches_reference_rule():
    from reagent_b200.training import CRRWeightFn

    adv = torch.tensor([-1.0, 0.0, 0.05, 2.0, 3.5])
    ind = CRRWeightFn(indicator_fn_threshold=0.05)
    assert torch.equal(ind.get_weight_from_advantage(adv), torch.tensor([0., 0., 1., 1., 1.]))
    ex = CRRWeightFn(exponent_beta=1.0, exponent_clamp=20.0)
    assert torch.equal(ex.get_weight_from_advantage(adv), torch.exp(adv).clamp(0.0, 20.0))
    assert torch.equal(ex.get_weight_from_advantage(adv),
                       V.crr_weight(adv, exponent_beta=1.0, exponent_clamp=20.0))
    with pytest.raises(AssertionError):
        CRRWeightFn()
    with pytest.raises(AssertionError):
        CRRWeightFn(indicator_fn_threshold=0.1, exponent_beta=1.0)
    with pytest.raises(AssertionError):
        CRRWeightFn(exponent_beta=1e-7)


def _nets(S=5, A=2, value=True):
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected

    actor = GaussianFullyConnectedActor(S, A, [8], ["relu"])
    q1 = FullyConnectedCritic(S, A, [8], ["relu"])
    q2 = FullyConnectedCritic(S, A, [8], ["relu"])
    v = FloatFeatureFullyConnected(S, 1, [8], ["relu"]) if value else None
    return actor, q1, q2, v


@pytest.mark.parametrize("name", ["sac_value_twin_alpha", "sac_value_fixed_alpha_odd"])
def test_sac_value_state_dict_keys_match_reference(name):
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.training import SACTrainer

    _, meta = G.load(name)
    S, A, sz, ac = meta["S"], meta["A"], meta["sizes"], meta["acts"]
    t = SACTrainer(GaussianFullyConnectedActor(S, A, sz, ac), FullyConnectedCritic(S, A, sz, ac),
                   FullyConnectedCritic(S, A, sz, ac), FloatFeatureFullyConnected(S, 1, sz, ac),
                   **({} if meta["learn_alpha"] else {"alpha_optimizer": None}))
    assert sorted(t.state_dict().keys()) == meta["state_dict_keys"]
    assert not hasattr(t, "q1_network_target")


def test_sac_value_optimizer_order():
    from reagent_b200.training import SACTrainer

    actor, q1, q2, v = _nets()
    t = SACTrainer(actor, q1, q2, v)
    opts = [o["optimizer"] for o in t.configure_optimizers()]
    assert len(opts) == 6  # q1, q2, actor, alpha, value, SoftUpdate(value target)
    assert [p.data_ptr() for p in opts[4].param_groups[0]["params"]] == \
        [p.data_ptr() for p in v.parameters()]


def test_sac_crr_construction_rules():
    from reagent_b200.training import CRRWeightFn, SACTrainer

    crr = CRRWeightFn(exponent_beta=1.0)
    actor, q1, q2, v = _nets()
    with pytest.raises(AssertionError):
        SACTrainer(actor, q1, q2, None, crr_config=crr)
    with pytest.raises(ValueError):
        SACTrainer(actor, q1, q2, v, crr_config=crr, backprop_through_log_prob=False)
    with pytest.raises(NotImplementedError):
        SACTrainer(actor, q1, q2, v, action_embedding_kld_weight=0.5)
    t = SACTrainer(actor, q1, q2, v, crr_config=crr)
    assert t.crr_config is crr


def test_value_builder_and_manager_fields():
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters
    from reagent_b200.model_managers import SAC
    from reagent_b200.net_builder import ValueFullyConnected

    state = NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS", mean=0.0, stddev=1.0)
        for i in range(3)})
    b = ValueFullyConnected(sizes=[64, 64], activations=["leaky_relu", "leaky_relu"])
    v = b.build_value_network(state)
    assert v.arena.dims == [3, 64, 64, 1]
    with pytest.raises(NotImplementedError):
        ValueFullyConnected(use_layer_norm=True).build_value_network(state)
    with pytest.raises(AssertionError):
        ValueFullyConnected(sizes=[4], activations=["relu", "relu"])
    m = SAC()
    assert m.value_net_builder is None and m.crr_config is None
    assert m.logged_action_uniform_prior and m.backprop_through_log_prob
