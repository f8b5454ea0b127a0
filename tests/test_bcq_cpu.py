"""Batch-constrained Q-learning without a GPU: the CPU oracle (oracle/bcq_oracle.py on oracle/td_oracle.py) pinned to
golden vectors of the unmodified reference DQNTrainer / BatchConstrainedDQN
(oracle/make_bcq_golden.py), and the constructor surface of DQNTrainer(imitator=, bcq=) and
BatchConstrainedDQN."""
import numpy as np
import pytest
import torch

from oracle import bcq_oracle as BO
from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import BCQ_DQN_CASES, _dqn_kwargs


def _imitator(arrays, meta):
    return G.oracle_net(arrays, "im", meta["imitator_acts"])


@pytest.mark.parametrize("name", BCQ_DQN_CASES)
def test_bcq_filter_oracle_matches_reference(name):
    """Filter values on state and next_state, the filtered next-action mask of update 0 and the
    masks the reference left behind in the batch (its in-place `*=`)."""
    arrays, meta = G.load(name)
    im = _imitator(arrays, meta)
    batch = G.batch_tensors(arrays)
    thr = meta["bcq"]
    keep_s, r_s = BO.bcq_filter(im, batch["state"], thr)
    keep_n, r_n = BO.bcq_filter(im, batch["next_state"], thr)
    assert G.rel_err(r_s, arrays["bcq.r_state"]) < 1e-6
    assert G.rel_err(r_n, arrays["bcq.r_next_state"]) < 1e-6
    # the goldens keep every r at least 1e-4 (relative) away from the threshold
    assert torch.equal(keep_n, torch.from_numpy(arrays["bcq.r_next_state"] >= thr).float())
    want_next = (batch["possible_next_actions_mask"] * keep_n).numpy()
    assert np.array_equal(want_next, arrays["bcq.next_mask0"])
    assert np.array_equal(want_next, arrays["after.possible_next_actions_mask"])
    assert np.array_equal((batch["possible_actions_mask"] * keep_s).numpy(),
                          arrays["after.possible_actions_mask"])
    # the filter does narrow the mask, and every non-terminal row keeps an action
    assert (want_next < arrays["batch.possible_next_actions_mask"]).any()
    nt = arrays["batch.not_terminal"].reshape(-1) > 0
    assert (want_next[nt].sum(1) >= 1).all()


@pytest.mark.parametrize("name", BCQ_DQN_CASES)
def test_bcq_dqn_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = _dqn_kwargs(meta, batch)
    kw.update(imitator=_imitator(arrays, meta), bcq_threshold=meta["bcq"])
    cpe = meta["cpe_metrics"] is not None
    if cpe:
        rn = G.oracle_net(arrays, "r0", acts, requires_grad=True)
        qc = G.oracle_net(arrays, "c0", acts, requires_grad=True)
        qct = G.oracle_net(arrays, "ct0", acts)
        adam_r = O.AdamState(O.net_params(rn), lr=meta["lr"])
        adam_c = O.AdamState(O.net_params(qc), lr=meta["lr"])
        ckw = dict(gamma=meta["gamma"], temperature=meta["temperature"], num_actions=meta["A"],
                   maxq=meta["maxq"], loss=meta["loss"], discount_src=kw.get("discount_src"),
                   imitator=kw["imitator"], bcq_threshold=meta["bcq"])
    for it in range(meta["n_updates"]):
        loss, grads, aux = BO.dqn_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            assert np.array_equal(aux["next_mask"].numpy(), arrays["bcq.next_mask0"])
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6
            assert G.rel_err(aux["all_q"], arrays["all_q0"]) < 1e-6
        if cpe:
            if it == 0:
                # the reference's CPE head sees the FILTERED mask (float32 batch mask, written
                # in place); with the unfiltered one the CPE q-value loss would differ
                unf = {k: v for k, v in ckw.items() if k not in ("imitator", "bcq_threshold")}
                _, cl_unfiltered, _ = O.dqn_cpe_losses(q, rn, qc, qct, batch, **unf)
                assert abs(float(cl_unfiltered) - arrays["cpe_losses"][0][1]) > 1e-4
            rl, cl, gr, gc = BO.dqn_cpe_update(q, rn, adam_r, qc, qct, adam_c, batch,
                                              tau=meta["tau"], **ckw)
            for got, want in ((rl, arrays["cpe_losses"][it][0]), (cl, arrays["cpe_losses"][it][1])):
                assert abs(got - want) <= 1e-6 * max(1.0, abs(want)), (it, got, want)
            if it == 0:
                for i, g in enumerate(gr):
                    assert G.rel_err(g, arrays[f"grad0r.{i}"]) < 1e-6
                for i, g in enumerate(gc):
                    assert G.rel_err(g, arrays[f"grad0c.{i}"]) < 1e-6
    nets = [(q, "qN"), (qt, "qtN")]
    if cpe:
        nets += [(rn, "rN"), (qc, "cN"), (qct, "ctN")]
    for net, prefix in nets:
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], b) < 1e-6, (prefix, i)


def test_bcq_model_oracle_matches_reference():
    """BatchConstrainedDQN.forward = q(s) + (-1e10) * (r < thr) (reagent/models/bcq.py:26-35)."""
    arrays, meta = G.load("bcq_model_forward")
    q = G.oracle_net(arrays, "q0", ["relu"] * len(meta["sizes"]) + ["linear"])
    im = G.oracle_net(arrays, "im", meta["imitator_acts"])
    x = torch.from_numpy(arrays["state"])
    keep, r = BO.bcq_filter(im, x, meta["thr"])
    assert G.rel_err(r, arrays["r"]) < 1e-6
    qv = O.mlp(q, x).detach()
    assert G.rel_err(qv, arrays["q_values"]) < 1e-6
    out = BO.model_forward(q, im, x, meta["thr"])
    want = torch.from_numpy(arrays["out"])
    dropped = keep == 0
    assert 0 < int(dropped.sum()) < dropped.numel()
    assert torch.equal(out[dropped], want[dropped])
    assert G.rel_err(out[~dropped], want[~dropped]) < 1e-6


# ---------------------------------------------------------------------------
# constructor surface
# ---------------------------------------------------------------------------
S, A = 8, 3


def _trainer(**kw):
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import DQNTrainer

    torch.manual_seed(0)
    q = FullyConnectedDQN(S, A, [16], ["relu"])
    cpe = kw.pop("cpe", False)
    nets = ()
    if cpe:
        rn, qc = FullyConnectedDQN(S, A, [16], ["relu"]), FullyConnectedDQN(S, A, [16], ["relu"])
        nets = (rn, qc, qc.get_target_network())
    return DQNTrainer(q, q.get_target_network(), *nets, actions=[str(i) for i in range(A)],
                      evaluation=EvaluationParameters(calc_cpe_in_training=cpe), **kw)


def _imitator_net(out=A):
    from reagent_b200.models import FullyConnectedNetwork

    return FullyConnectedNetwork([S, 16, out], ["relu", "linear"])


def test_bcq_constructor_errors():
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training.dqn_trainer import BCQConfig

    with pytest.raises(NotImplementedError, match="FullyConnectedNetwork"):
        _trainer(imitator=torch.nn.Linear(S, A), bcq=BCQConfig(0.3))
    with pytest.raises(NotImplementedError, match="FullyConnectedNetwork"):
        _trainer(imitator=lambda x: np.ones((x.shape[0], A)), bcq=BCQConfig(0.3))  # scikit-style
    with pytest.raises(NotImplementedError, match="FullyConnectedNetwork"):
        _trainer(imitator=FullyConnectedDQN(S, A, [16], ["relu"]), bcq=BCQConfig(0.3))
    with pytest.raises(ValueError, match="4 outputs"):
        _trainer(imitator=_imitator_net(4), bcq=BCQConfig(0.3))
    with pytest.raises(ValueError, match="needs an imitator"):
        _trainer(bcq=BCQConfig(0.3))
    with pytest.raises(ValueError, match="maxq_learning=True"):
        _trainer(imitator=_imitator_net(), bcq=BCQConfig(0.3), rl=RLParameters(maxq_learning=False))
    # an imitator without bcq is accepted and ignored, as in the reference
    t = _trainer(imitator=_imitator_net())
    assert not t.bcq and not hasattr(t, "bcq_imitator")


@pytest.mark.parametrize("cpe", [False, True])
def test_bcq_optimizers_leave_the_imitator_alone(cpe):
    from reagent_b200.optimizer import FusedAdam, SoftUpdate
    from reagent_b200.training.dqn_trainer import BCQConfig

    im = _imitator_net()
    t = _trainer(imitator=im, bcq=BCQConfig(0.25), cpe=cpe)
    assert t.bcq and t.bcq_drop_threshold == 0.25 and t.bcq_imitator is im
    assert dict(t.named_children())["bcq_imitator"] is im  # a registered sub-module
    want = [FusedAdam, FusedAdam, FusedAdam, SoftUpdate] if cpe else [FusedAdam, SoftUpdate]
    opts = t.optimizers()
    assert [type(o) for o in opts] == want
    im_ids = {id(p) for p in im.parameters()}
    for o in opts:
        for g in o.param_groups:
            assert not im_ids & {id(p) for p in g["params"]}
    base = _trainer(cpe=cpe)
    assert ([len(g["params"]) for o in opts for g in o.param_groups]
            == [len(g["params"]) for o in base.optimizers() for g in o.param_groups])


def test_bcq_cpe_mask_follows_the_reference_aliasing_rule():
    """CPE reads the filtered next-action mask exactly when the batch mask is float32 (the
    reference's `.float()` then returns the batch tensor, which its `*=` filters in place)."""
    from reagent_b200.core import types as rlt
    from reagent_b200.training.dqn_trainer import BCQConfig

    t = _trainer(imitator=_imitator_net(), bcq=BCQConfig(0.3), cpe=True)
    filtered = torch.zeros(2, A)
    t.bcq_next_actions_mask = filtered

    def batch(mask):
        return rlt.DiscreteDqnInput(
            state=rlt.FeatureData(torch.zeros(2, S)), next_state=rlt.FeatureData(torch.zeros(2, S)),
            action=torch.zeros(2, A), next_action=torch.zeros(2, A), reward=torch.zeros(2, 1),
            not_terminal=torch.ones(2, 1), possible_actions_mask=torch.ones(2, A),
            possible_next_actions_mask=mask, step=None, time_diff=None, extras=rlt.ExtraData())

    assert t._cpe_next_mask(batch(torch.ones(2, A))) is filtered
    assert t._cpe_next_mask(batch(torch.ones(2, A, dtype=torch.bool))) is None
    assert t._cpe_next_mask(batch(torch.ones(2, A, dtype=torch.float64))) is None
    assert _trainer(cpe=True)._cpe_next_mask(batch(torch.ones(2, A))) is None


def test_batch_constrained_dqn_constructs_with_the_reference_state_dict():
    from reagent_b200.models import BatchConstrainedDQN, FullyConnectedDQN, FullyConnectedNetwork

    arrays, meta = G.load("bcq_model_forward")
    q = FullyConnectedDQN(meta["S"], meta["A"], meta["sizes"], ["relu"] * len(meta["sizes"]))
    im = FullyConnectedNetwork([meta["S"]] + meta["imitator_sizes"] + [meta["A"]],
                               meta["imitator_acts"])
    m = BatchConstrainedDQN(meta["S"], q, im, meta["thr"])
    assert list(m.state_dict().keys()) == meta["state_dict_keys"]
    assert m.invalid_action_penalty == -1e10 and m.bcq_drop_threshold == meta["thr"]
    assert m.input_prototype().float_features.shape == (1, meta["S"])
    with pytest.raises(AssertionError):
        BatchConstrainedDQN(0, q, im, 0.3)
    with pytest.raises(NotImplementedError, match="FullyConnectedNetwork"):
        BatchConstrainedDQN(meta["S"], q, torch.nn.Linear(meta["S"], meta["A"]), 0.3)


def test_bcq_filter_rejects_bad_arguments():
    """Argument checks of the C entry point run before any launch (no GPU needed): the pointer
    values below are never dereferenced."""
    from reagent_b200 import _lib

    lib = _lib.lib()
    p = 4096
    bad = [  # logits, B, A, thr, mask_in, mask_out, q_in, q_out
        (p, 0, 4, 0.3, None, p, None, None),
        (p, 4, 0, 0.3, None, p, None, None),
        (p, 4, 1025, 0.3, None, p, None, None),
        (None, 4, 4, 0.3, None, p, None, None),
        (p, 4, 4, float("nan"), None, p, None, None),
        (p, 4, 4, 0.3, None, None, None, None),   # no output
        (p, 4, 4, 0.3, None, p, p, p),            # both outputs
        (p, 4, 4, 0.3, None, None, None, p),      # q_out without q_in
        (p, 4, 4, 0.3, p, None, p, p),            # mask_in in model mode
        (p, 4, 4, 0.3, None, p, p, None),         # q_in in trainer mode
    ]
    for args in bad:
        assert lib.rb200_bcq_filter(*args, None) == -1, args  # RB200_E_INVALID
        assert lib.rb200_last_error().startswith(b"rb200_bcq_filter"), args
