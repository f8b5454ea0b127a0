"""Discrete CRR without a GPU: the plain-torch restatement (oracle/crr_oracle.py) against every
golden of the unmodified reference, the structure the goldens record, constructor and manager
defaults and the refusals."""
import glob
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import crr_oracle as CO
from oracle import td_oracle as O
from oracle.adamw_oracle import AdamWState
from oracle.ref_harness import reference_available
from tests import golden_util as G
from tests.golden_cases import (CRR_CASES, check_grads, check_losses, check_params, initial_tensors,
                                net_names, noise_of)
from tests.golden_util import TOL


def _acts(meta, name):
    return meta["acts"] + ["tanh" if name.startswith("actor") else "linear"]


def oracle_net(arrays, meta, name):
    if not meta["compact"]:
        return G.oracle_net(arrays, name + "0", _acts(meta, name), requires_grad=True)
    ts = initial_tensors(arrays, meta, name)
    return {"W": [t.requires_grad_(True) for t in ts[0::2]],
            "b": [t.requires_grad_(True) for t in ts[1::2]], "act": _acts(meta, name)}


def update_kwargs(meta):
    boost = None
    if meta["boost"]:
        boost = torch.zeros(1, meta["A"])
        for k, v in meta["boost"].items():
            boost[0, int(k)] = v
    return dict(gamma=meta["gamma"], tau=meta["tau"], use_target_actor=meta["use_target_actor"],
                delayed_policy_update=meta["delayed_policy_update"], beta=meta["beta"],
                entropy_coeff=meta["entropy_coeff"], clip_limit=meta["clip_limit"],
                max_weight=meta["max_weight"], reward_boost=boost,
                temperature=meta["temperature"])


@pytest.mark.parametrize("name", CRR_CASES)
def test_crr_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    src, tgt = net_names(meta)
    nets = {n: oracle_net(arrays, meta, n) for n in src + tgt}
    if meta["optimizer"] == "AdamW":
        adam = lambda ps: AdamWState(ps, lr=meta["lr"], **meta["opt_kw"])  # noqa: E731
    else:
        adam = lambda ps: O.AdamState(ps, lr=meta["lr"])  # noqa: E731
    st = CO.CrrState(nets["actor"], nets["actor_t"], nets["q1"], nets["q1_t"], nets.get("q2"),
                     nets.get("q2_t"), nets.get("r"), nets.get("c"), nets.get("ct"),
                     make_adam_q=adam, make_adam_actor=adam)
    batch = G.batch_tensors(arrays)
    for it in range(meta["n_updates"]):
        losses, grads, weight = CO.crr_update(
            st, batch, it, noise_next=noise_of(arrays, it, "next"),
            noise_cur=noise_of(arrays, it, "cur"), **update_kwargs(meta))
        check_losses(arrays, it, losses)
        if it == 0:
            for oi, g in enumerate(grads):
                check_grads(arrays, meta, oi, g)
            assert G.rel_err(weight.view(-1), arrays["weight0"]) < TOL
    for n in src + tgt:
        check_params(arrays, meta, n, [p.detach() for p in O.net_params(nets[n])])


def _tiny_trainer(**kw):
    from reagent_b200.models import FullyConnectedActor, FullyConnectedDQN
    from reagent_b200.training import DiscreteCRRTrainer

    nets = dict(actor_network=FullyConnectedActor(5, 3, [8], ["relu"]),
                q1_network=FullyConnectedDQN(5, 3, [8], ["relu"]), reward_network=None)
    nets.update({k: v for k, v in kw.items() if k.endswith("network")})
    rest = {k: v for k, v in kw.items() if not k.endswith("network")}
    rest.setdefault("actions", ["a", "b", "c"])
    return DiscreteCRRTrainer(
        actor_network_target=nets["actor_network"].get_target_network()
        if hasattr(nets["actor_network"], "get_target_network") else None,
        q1_network_target=nets["q1_network"].get_target_network()
        if hasattr(nets["q1_network"], "get_target_network") else None, **nets, **rest)


def test_constructor_defaults_are_the_references():
    from reagent_b200.training import DiscreteCRRTrainer

    p = inspect.signature(DiscreteCRRTrainer.__init__).parameters
    want = dict(q2_network=None, q2_network_target=None, q_network_cpe=None,
                q_network_cpe_target=None, metrics_to_score=None, double_q_learning=True,
                use_target_actor=False, delayed_policy_update=1, beta=1.0, entropy_coeff=0.0,
                clip_limit=10.0, max_weight=20.0)
    for k, v in want.items():
        assert p[k].default == v, k
    assert list(p)[1:6] == ["actor_network", "actor_network_target", "q1_network",
                            "q1_network_target", "reward_network"]
    if reference_available():
        from oracle.ref_harness import ref

        rp = inspect.signature(
            ref("reagent.training.discrete_crr_trainer").DiscreteCRRTrainer.__init__).parameters
        assert list(rp) == list(p)


@pytest.mark.parametrize("name", ["crr_twin_default", "crr_single_target_actor", "crr_cpe_boost"])
def test_optimizer_order_matches_the_goldens_structure(name):
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import SoftUpdate

    _, meta = G.load(name)
    kw = {}
    if meta["twin"]:
        kw["q2_network"] = FullyConnectedDQN(5, 3, [8], ["relu"])
        kw["q2_network_target"] = kw["q2_network"].get_target_network()
    cpe = meta["cpe_metrics"] is not None
    if cpe:
        kw["reward_network"] = FullyConnectedDQN(5, 6, [8], ["relu"])
        kw["q_network_cpe"] = FullyConnectedDQN(5, 6, [8], ["relu"])
        kw["q_network_cpe_target"] = kw["q_network_cpe"].get_target_network()
        kw["metrics_to_score"] = meta["cpe_metrics"]
    # q2_network_target / q_network_cpe_target do not end in "network": they pass through `rest`
    t = _tiny_trainer(evaluation=EvaluationParameters(calc_cpe_in_training=cpe), **kw)
    owner = {}
    for k, net in (("q1", t.q1_network), ("q2", t.q2_network), ("actor", t.actor_network),
                   ("r", t.reward_network), ("c", t.q_network_cpe),
                   ("q1_t", t.q1_network_target), ("q2_t", t.q2_network_target),
                   ("actor_t", t.actor_network_target), ("ct", t.q_network_cpe_target)):
        if net is not None:
            owner.update({id(p): k for p in net.parameters()})
    opts = t.optimizers()
    assert len(opts) == meta["n_yields"]
    assert [owner[id(o.param_groups[0]["params"][0])] for o in opts[:-1]] == meta["optimizers"]
    assert isinstance(opts[-1], SoftUpdate)
    su = opts[-1].param_groups[0]["params"]
    assert list(dict.fromkeys(owner[id(p)] for p in su[:len(su) // 2])) == meta["soft_update_targets"]
    assert t.q_network is t.q1_network


def test_manager_and_builder_defaults():
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.model_managers import DiscreteCRR
    from reagent_b200.net_builder import DiscreteActorFullyConnected, Dueling, FullyConnected

    b = DiscreteActorFullyConnected()
    assert (b.sizes, b.activations, b.action_activation, b.exploration_variance,
            b.use_batch_norm) == ([128, 64], ["relu", "relu"], "tanh", None, False)
    m = DiscreteCRR(actions=["0", "1"])
    assert isinstance(m.actor_net_builder, DiscreteActorFullyConnected)
    assert isinstance(m.critic_net_builder, Dueling)
    assert isinstance(m.cpe_net_builder, FullyConnected)
    assert m.eval_parameters == EvaluationParameters() and m.rl == RLParameters()
    assert (m.double_q_learning, m.use_target_actor, m.delayed_policy_update, m.beta,
            m.entropy_coeff, m.clip_limit, m.max_weight) == (True, False, 1, 1.0, 0.0, 10.0, 20.0)
    assert m.action_names == ["0", "1"] and m.rl_parameters is m.rl
    with pytest.raises(AssertionError, match="at least 2 actions"):
        DiscreteCRR(actions=["only"])
    with pytest.raises(RuntimeError, match="CUDA only"):
        m.build_trainer({}, use_gpu=False)
    with pytest.raises(NotImplementedError, match="serving"):
        m.create_policy(None, serving=True)
    with pytest.raises(NotImplementedError, match="layer norm"):
        DiscreteActorFullyConnected(use_layer_norm=True)
    with pytest.raises(NotImplementedError):
        DiscreteActorFullyConnected(use_batch_norm=True).build_actor(_norm(4), 2)


def _norm(n):
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters

    return NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS", mean=0.0, stddev=1.0)
        for i in range(n)})


def test_networks_the_fused_kernels_cannot_run_are_refused():
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected

    with pytest.raises(NotImplementedError, match="FullyConnectedActor"):
        _tiny_trainer(actor_network=FullyConnectedDQN(5, 3, [8], ["relu"]))
    with pytest.raises(NotImplementedError, match="without atoms"):
        _tiny_trainer(q1_network=FullyConnectedDQN(5, 3, [8], ["relu"], num_atoms=5))
    with pytest.raises(NotImplementedError, match="q1_network must be"):
        _tiny_trainer(q1_network=FloatFeatureFullyConnected(5, 3, [8], ["relu"]))
    with pytest.raises(ValueError, match="3 actions"):
        _tiny_trainer(q1_network=FullyConnectedDQN(5, 4, [8], ["relu"]))


def test_exports():
    import reagent_b200.model_managers as mm
    import reagent_b200.net_builder as nb
    import reagent_b200.training as tr

    assert tr.DiscreteCRRTrainer.__mro__[1].__name__ == "DQNTrainerBaseLightning"
    assert hasattr(mm, "DiscreteCRR") and hasattr(nb, "DiscreteActorFullyConnected")
    for m in ("train_step_gen", "train_batch", "validation_step", "configure_optimizers",
              "get_detached_model_outputs"):
        assert callable(getattr(tr.DiscreteCRRTrainer, m))


def test_every_committed_crr_golden_is_a_known_case():
    names = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G.GOLDEN, "crr_*.npz")))
    assert names == sorted(CRR_CASES)


@pytest.mark.skipif(not reference_available(), reason="the reference checkout is not here")
@pytest.mark.parametrize("name", [n for n in CRR_CASES if n != "crr_cartpole_manager"])
def test_goldens_regenerate_identically_from_the_reference(name, tmp_path, monkeypatch):
    """Bit for bit for the small cases; the [1024, 1024] case's GEMMs may sum in another order
    with another thread count, and test_crr_oracle_matches_reference holds it to 1e-5."""
    import oracle.make_golden as MG
    from oracle import make_crr_golden

    monkeypatch.setattr(MG, "GOLDEN", str(tmp_path))
    make_crr_golden.main({name})
    new = np.load(os.path.join(str(tmp_path), name + ".npz"))
    old = np.load(os.path.join(G.GOLDEN, name + ".npz"))
    assert sorted(new.files) == sorted(old.files)
    for k in old.files:
        assert np.array_equal(new[k], old[k], equal_nan=True), k
