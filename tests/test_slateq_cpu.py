"""SlateQ without a GPU: the float64 oracle (oracle/slateq_oracle.py) against every SlateQ golden
of the unmodified reference (oracle/make_slateq_golden.py) and, where the reference is present,
against the reference itself; the trainer's constructor, optimizer order and batch type; the
input maker it selects; and the SlateQ manager built from each RecSim configuration's fields."""
import inspect

import numpy as np
import pytest
import torch

from oracle import slateq_oracle as SO
from oracle.ref_harness import reference_available
from oracle.td_oracle import AdamState, net_params
from tests import golden_util as G
from tests import slateq_cases as SC


@pytest.mark.parametrize("name", SC.TRAINER_CASES)
def test_oracle_matches_the_goldens(name):
    arrays, meta = G.load(name)
    q, qt = SC.oracle_nets(arrays, meta)
    adam = AdamState(net_params(q), lr=meta["lr"])
    kw = SC.oracle_kwargs(meta)
    for it in range(meta["n_updates"]):
        b = SC.batch(arrays, it)
        loss, _, nxt = SO.slateq_update(q, qt, adam, b, tau=meta["tau"], **kw)
        want = arrays["losses"][it]
        assert abs(loss - want) <= 1e-5 * max(1.0, abs(want)), (it, loss, want)
        if not meta["maxq"]:
            assert np.array_equal(nxt.numpy(), arrays[f"batch{it}.next_action_after"])
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = net_params(net)
        for i, (w, bias) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-5 and G.rel_err(ps[2 * i + 1], bias) < 1e-5, (prefix, i)


def test_goldens_cover_terminal_rows_and_the_null_slot():
    for name in SC.TRAINER_CASES:
        arrays, meta = G.load(name)
        bs = [SC.batch(arrays, it) for it in range(meta["n_updates"])]
        assert any((~b["not_terminal"]).any() for b in bs), name
        # the null slot (index slate_size) is appended to every slate
        assert all((b["action"][:, -1] == meta["slate_size"]).all() for b in bs), name
        assert any((b["reward_mask"][:, -1] & ~b["reward_mask"][:, :-1].any(1)).any() for b in bs), name


@pytest.mark.skipif(not reference_available(), reason="the reference is not present")
@pytest.mark.parametrize("maxq,single,norm_next", [(False, True, False), (True, True, False),
                                                   (False, False, True), (True, False, False)])
def test_oracle_matches_the_reference(maxq, single, norm_next):
    """One update of the reference trainer on a fresh odd-shaped batch with partial masks."""
    from oracle.make_slateq_golden import make_batch, ref_batch
    from oracle.ref_harness import ref, run_update

    rlt = ref("reagent.core.types")
    params = ref("reagent.core.parameters")
    critic = ref("reagent.models.critic")
    tr = ref("reagent.training.slate_q_trainer")
    union = ref("reagent.optimizer.union")
    torch.manual_seed(3)
    rq = critic.FullyConnectedCritic(6, 4, [16, 8], ["relu", "leaky_relu"])
    rqt = rq.get_target_network()
    q = SO.to64({"W": [s[0].weight for s in rq.fc.dnn], "b": [s[0].bias for s in rq.fc.dnn],
                 "act": ["relu", "leaky_relu", "linear"]}, requires_grad=True)
    qt = SO.to64(q)
    norm = "norm_by_next_slate_size" if norm_next else "norm_by_current_slate_size"
    trainer = tr.SlateQTrainer(
        rq, rqt, 3, rl=params.RLParameters(gamma=0.8, target_update_rate=0.3, maxq_learning=maxq),
        optimizer=union.Optimizer__Union(Adam=union.classes["Adam"](lr=0.01)),
        slate_opt_parameters=params.SlateOptParameters(method=params.SlateOptMethod.TOP_K),
        discount_time_scale=1.5, single_selection=single,
        next_slate_value_norm_method=tr.NextSlateValueNormMethod(norm),
        evaluation=params.EvaluationParameters(calc_cpe_in_training=False))
    b = make_batch(29, 9, 3, 6, 4, torch.Generator().manual_seed(5), partial_masks=not maxq,
                   p_term=0.3, time_diff=True)
    rb = ref_batch(rlt, {k: v.clone() for k, v in b.items()})
    want = run_update(trainer, rb, 0)[0]
    got, _, nxt = SO.slateq_update(q, qt, AdamState(net_params(q), lr=0.01), b, tau=0.3,
                                   gamma=0.8, slate_size=3, maxq=maxq, single_selection=single,
                                   norm_next=norm_next, time_scale=1.5)
    assert abs(got - want) <= 1e-5 * max(1.0, abs(want))
    if not maxq:
        assert torch.equal(nxt, rb.next_action)
    for i, seq in enumerate(rq.fc.dnn):
        assert G.rel_err(q["W"][i], seq[0].weight) < 1e-5
        assert G.rel_err(qt["W"][i], rqt.fc.dnn[i][0].weight) < 1e-5


def test_constructor_defaults_are_the_references():
    from reagent_b200.training import NextSlateValueNormMethod, SlateQTrainer

    p = inspect.signature(SlateQTrainer.__init__).parameters
    assert list(p) == ["self", "q_network", "q_network_target", "slate_size", "rl", "optimizer",
                       "slate_opt_parameters", "discount_time_scale", "single_selection",
                       "next_slate_value_norm_method", "minibatch_size", "evaluation"]
    want = dict(slate_opt_parameters=None, discount_time_scale=None, single_selection=True,
                next_slate_value_norm_method=NextSlateValueNormMethod.NORM_BY_CURRENT_SLATE_SIZE,
                minibatch_size=1024)
    for k, v in want.items():
        assert p[k].default == v, k
    if reference_available():
        from oracle.ref_harness import ref

        rp = inspect.signature(ref("reagent.training.slate_q_trainer").SlateQTrainer.__init__).parameters
        assert list(rp) == list(p)


def _trainer(**kw):
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.training import SlateQTrainer

    q = FullyConnectedCritic(5, 3, [8], ["relu"])
    return SlateQTrainer(q, q.get_target_network(), 2, **kw)


def test_defaults_and_optimizer_order():
    from reagent_b200.core import types as rlt
    from reagent_b200.gym.preprocessors.trainer_preprocessor import (REPLAY_BUFFER_MAKER_MAP,
                                                                     SlateQInputMaker)
    from reagent_b200.optimizer import FusedAdam, SoftUpdate

    t = _trainer()
    assert t.rl_parameters.maxq_learning is False
    assert t.gamma == 0.9 and t.tau == 0.001
    opts = [o["optimizer"] for o in t.configure_optimizers()]
    assert [type(o) for o in opts] == [FusedAdam, SoftUpdate]
    ann = inspect.signature(t.train_step_gen).parameters["training_batch"].annotation
    assert ann is rlt.SlateQInput
    assert REPLAY_BUFFER_MAKER_MAP[ann] is SlateQInputMaker


def test_maxq_needs_top_k_slate_optimisation():
    """_get_maxq_next_action: max-Q without slate_opt_parameters fails the reference's assert;
    GREEDY / EXACT are not implemented.  Both are refused before anything touches a device."""
    from reagent_b200.core.parameters import RLParameters, SlateOptMethod, SlateOptParameters

    arrays, _ = G.load("slateq_odd_shapes")
    from reagent_b200.core import types as rlt

    batch = SC.slateq_input(SC.batch(arrays, 0), rlt)
    with pytest.raises(AssertionError):
        _trainer(rl=RLParameters(maxq_learning=True)).train_batch(batch)
    for m in (SlateOptMethod.GREEDY, SlateOptMethod.EXACT):
        t = _trainer(rl=RLParameters(maxq_learning=True),
                     slate_opt_parameters=SlateOptParameters(method=m))
        with pytest.raises(NotImplementedError):
            t.train_batch(batch)


@pytest.mark.parametrize("yaml_name", sorted(SC.RECSIM_YAML.values()))
def test_manager_fields_of_each_recsim_configuration(yaml_name):
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.training import NextSlateValueNormMethod, SlateQTrainer

    m = SC.recsim_manager(yaml_name)
    assert m.eval_parameters.calc_cpe_in_training is False
    q = FullyConnectedCritic(20, 20, m.net_builder.sizes, m.net_builder.activations)
    t = SlateQTrainer(q, q.get_target_network(), m.slate_size, **m.trainer_param.asdict())
    assert t.slate_size == 3
    assert t.rl_parameters.maxq_learning == yaml_name.endswith("_maxq_topk.yaml")
    assert t.slate_opt_parameters is None
    assert t.single_selection == ("_multi_selection" not in yaml_name)
    assert isinstance(t.next_slate_value_norm_method, NextSlateValueNormMethod)
    with pytest.raises(RuntimeError):
        m.build_trainer({}, use_gpu=False)
    with pytest.raises(NotImplementedError):
        m.create_policy(t, serving=True)


def test_manager_needs_slate_size_and_candidates():
    from reagent_b200.model_managers import SlateQ

    with pytest.raises(AssertionError):
        SlateQ(num_candidates=10)
    with pytest.raises(AssertionError):
        SlateQ(slate_size=3)


def test_doc_list_select_slate_and_feature_data_default():
    from reagent_b200.core import types as rlt

    f = torch.arange(2 * 4 * 3, dtype=torch.float32).view(2, 4, 3)
    d = rlt.DocList(f)
    assert d.mask.dtype == torch.bool and d.mask.all() and (d.value == 1).all()
    s = d.select_slate(torch.tensor([[3, 0], [1, 1]]))
    assert torch.equal(s.float_features[0, 0], f[0, 3]) and torch.equal(s.float_features[1, 1], f[1, 1])
    assert s.as_feature_data().float_features.shape == (4, 3)
    fd = rlt.FeatureData(torch.zeros(2, 5))
    assert fd.candidate_docs is None and fd.float().candidate_docs is None
    fd2 = rlt.FeatureData(torch.zeros(2, 5), candidate_docs=d).to(torch.float64)
    assert fd2.candidate_docs.float_features.dtype == torch.float64
