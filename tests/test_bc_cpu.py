"""Behavioral cloning without a GPU: the CPU oracle (oracle/bc_oracle.py) pinned to golden vectors
of the unmodified reference BehavioralCloningTrainer (oracle/make_bc_golden.py), the offline
BCQ scenario of tests/test_bc_gpu.py on the oracle (where its thresholds come from), and the
constructor, input-check and C-ABI surface of BehavioralCloningTrainer."""
import inspect

import pytest
import torch

from oracle import bc_oracle as BC
from oracle import bcq_oracle as BO
from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import (BC_CASES, E2E, E2E_MAX_KEPT, E2E_MIN_BEHAVIOUR_KEPT, e2e_data,
                                e2e_metrics, golden_batch)


@pytest.mark.parametrize("name", BC_CASES)
def test_bc_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    net = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    adam = O.AdamState(O.net_params(net), lr=meta["lr"])
    for it in range(meta["n_updates"]):
        b = golden_batch(arrays, f"batch{it}")
        # the goldens' labels are rows of an involutive permutation: dim 0 and dim 1 agree
        assert torch.equal(b["action"].max(dim=0)[1], b["action"].argmax(dim=1))
        loss, grads, logits = BC.bc_update(net, adam, b)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it])), it
        assert G.rel_err(logits, arrays[f"logits{it}"]) < 1e-6
        for i, g in enumerate(grads):
            assert G.rel_err(g, arrays[f"grad{it}.{i}"]) < 1e-6, (it, i)
        for i, (w, bb) in enumerate(G.net_pairs(arrays, f"q{it + 1}")):
            assert G.rel_err(net["W"][i].detach(), w) < 1e-6, (it, i)
            assert G.rel_err(net["b"][i].detach(), bb) < 1e-6, (it, i)
    val, _ = BC.bc_loss(net, golden_batch(arrays, "val"))
    assert abs(float(val) - float(arrays["val_loss"])) <= 1e-6 * max(1.0, float(arrays["val_loss"]))


def test_bc_oracle_labels_each_row_with_its_own_action():
    """Off the goldens' inputs (B != A, or a label permutation that is not an involution) the
    reference's dim-0 labels raise or point at another row; this library's are per row."""
    g = torch.Generator().manual_seed(0)
    net = O.make_net([5, 8, 4], ["relu", "linear"], g)
    action = torch.nn.functional.one_hot(torch.tensor([1, 2, 3, 0]), 4).float()  # a 4-cycle
    b = dict(state=torch.randn(4, 5, generator=g), action=action, possible_actions_mask=torch.ones(4, 4))
    assert action.max(dim=0)[1].tolist() == [3, 0, 1, 2]
    loss, logits = BC.bc_loss(net, b)
    want = -torch.log_softmax(logits, dim=1)[torch.arange(4), torch.tensor([1, 2, 3, 0])].mean()
    assert float(loss) == pytest.approx(float(want), rel=1e-6)


# ---------------------------------------------------------------------------
# offline BCQ scenario: logged data from a deterministic behaviour rule -> BC -> BCQ filter
# ---------------------------------------------------------------------------


def test_offline_bcq_scenario_on_the_oracle():
    Wb, batches, held_out = e2e_data()
    g = torch.Generator().manual_seed(1)
    S, A = E2E["S"], E2E["A"]
    net = O.make_net([S] + E2E["sizes"] + [A], ["relu", "relu", "linear"], g)
    net = O.clone_net(net, requires_grad=True)
    adam = O.AdamState(O.net_params(net), lr=E2E["lr"])
    for b in batches:
        BC.bc_update(net, adam, b)
    keep, _ = BO.bcq_filter(net, held_out, E2E["thr"])
    kept_beh, kept = e2e_metrics(keep, Wb, held_out)
    print(f"offline BCQ on the oracle: behaviour action kept on {kept_beh:.4f} of the rows, "
          f"{kept:.4f} of all pairs kept")
    assert kept_beh >= E2E_MIN_BEHAVIOUR_KEPT, kept_beh
    assert kept <= E2E_MAX_KEPT, kept


# ---------------------------------------------------------------------------
# constructor, optimizer, input checks, C ABI
# ---------------------------------------------------------------------------
def _trainer(**kw):
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import BehavioralCloningTrainer

    return BehavioralCloningTrainer(FullyConnectedDQN(8, 4, [7, 6, 5], ["relu"] * 3), **kw)


def test_bc_constructor_and_optimizer():
    from reagent_b200.core import types as rlt
    from reagent_b200.optimizer import FusedAdam, Optimizer__Union

    t = _trainer()
    opts = t.optimizers()
    assert [type(o) for o in opts] == [FusedAdam]
    assert [id(p) for p in opts[0].param_groups[0]["params"]] == [id(p) for p in t.bc_net.parameters()]
    assert opts[0].param_groups[0]["lr"] == 1e-3  # Optimizer__Union.default(): Adam(lr=1e-3)
    assert _trainer(optimizer=Optimizer__Union.default(lr=0.05)).optimizers()[0].param_groups[0]["lr"] == 0.05
    sig = inspect.signature(t.train_step_gen)
    assert sig.parameters["training_batch"].annotation is rlt.BehavioralCloningModelInput
    assert t._training_batch_type is rlt.BehavioralCloningModelInput
    assert dict(t.named_children())["bc_net"] is t.bc_net


def test_bc_rejects_other_networks():
    from reagent_b200.models import DuelingQNetwork, FullyConnectedDQN, FullyConnectedNetwork
    from reagent_b200.training import BehavioralCloningTrainer

    for net in (torch.nn.Linear(8, 4), FullyConnectedNetwork([8, 16, 4], ["relu", "linear"]),
                FullyConnectedDQN(8, 4, [16], ["relu"], num_atoms=5),
                DuelingQNetwork.make_fully_connected(8, 4, [16, 8], ["relu", "relu"])):
        with pytest.raises(NotImplementedError, match="FullyConnectedDQN"):
            BehavioralCloningTrainer(net)


def test_behavioral_cloning_model_input():
    from reagent_b200.core import types as rlt

    d = dict(state=torch.randn(3, 8), action=torch.eye(3, 4), possible_actions_mask=torch.ones(3, 4))
    b = rlt.BehavioralCloningModelInput.from_dict(d)
    assert b.state.float_features is d["state"] and b.action is d["action"]
    assert b.possible_actions_mask is d["possible_actions_mask"] and b.batch_size() == 3
    d.pop("possible_actions_mask")
    assert rlt.BehavioralCloningModelInput.from_dict(d).possible_actions_mask is None


def _bc_batch(action, mask):
    from reagent_b200.core import types as rlt

    return rlt.BehavioralCloningModelInput(rlt.FeatureData(torch.randn(action.shape[0], 8)),
                                           action, mask)


@pytest.mark.parametrize("action, mask, exc", [
    (torch.tensor([1, 0, 0, 0]), torch.ones(4), TypeError),               # 1-D labels
    (torch.tensor([[1, 0, 0, 0]]), torch.ones(1, 4), TypeError),          # a single row
    (torch.eye(4), None, TypeError),                                      # no mask
    (torch.eye(4), torch.ones(4, 4) - torch.eye(4), AssertionError),      # labels masked out
    (torch.eye(4), torch.tensor([[1, 1, 0, 0]] * 4).float(), AssertionError),
])
def test_bc_check_input_errors(action, mask, exc):
    """The reference's _check_input: raised by train_step_gen and validation_step before any
    launch (so no GPU is needed)."""
    t = _trainer()
    with pytest.raises(exc):
        next(t.train_step_gen(_bc_batch(action, mask), 0))
    with pytest.raises(exc):
        t.validation_step(_bc_batch(action, mask), 0)


def test_bc_xent_head_rejects_bad_arguments():
    """Argument checks of the C entry point run before any launch (no GPU needed): the pointer
    values below are never dereferenced."""
    from reagent_b200 import _lib

    lib = _lib.lib()
    p = 4096

    def args(**kw):
        a = _lib.BcXentArgsT()
        a.batch, a.num_actions = 4, 4
        a.logits = a.labels = a.mask = a.dz = a.loss_partials = a.loss = a.tile_counter = p
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    assert lib.rb200_bc_xent_head(None, None) == -1
    bad = [dict(batch=0), dict(batch=-3), dict(num_actions=0), dict(num_actions=1025)]
    bad += [{k: None} for k in ("logits", "labels", "mask", "loss_partials", "loss", "tile_counter")]
    for kw in bad:
        assert lib.rb200_bc_xent_head(args(**kw), None) == -1, kw  # RB200_E_INVALID
        assert lib.rb200_last_error().startswith(b"rb200_bc_xent_head"), kw


def test_bc_needs_a_gpu_batch():
    from reagent_b200 import _lib

    with pytest.raises(_lib.Rb200Error):
        _trainer().train_batch(_bc_batch(torch.eye(4), torch.ones(4, 4)))
