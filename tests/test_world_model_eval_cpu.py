"""World-model evaluators without a GPU: the fp64 oracle against the reference's goldens, the
feature grouping and variant table, input validation, and the constructors."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import world_model_eval_oracle as wo  # noqa: E402
from oracle.ref_harness import reference_available  # noqa: E402
from tests.golden_util import load  # noqa: E402
from tests.world_model_eval_cases import (CASES, TOL, batch_of, cfg_of,  # noqa: E402
                                          importance_of, params64, sensitivity_tol)

from reagent_b200 import _lib  # noqa: E402
from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import MDNRNNTrainerParameters  # noqa: E402
from reagent_b200.evaluation import (FeatureImportanceEvaluator,  # noqa: E402
                                     FeatureSensitivityEvaluator, LossEvaluator)
from reagent_b200.evaluation.world_model_evaluator import (feature_groups,  # noqa: E402
                                                           importance_variants)
from reagent_b200.models import MemoryNetwork  # noqa: E402
from reagent_b200.training import MDNRNNTrainer  # noqa: E402


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_golden(name):
    arrays, meta = load(name)
    imp = importance_of(arrays, meta)
    want = torch.from_numpy(arrays["losses"])
    assert imp["losses"].shape == want.shape
    assert torch.all((imp["losses"] - want).abs() <= TOL * want.abs()), (imp["losses"], want)
    for v, f in enumerate(imp["fills"][1:], start=1):
        g = torch.from_numpy(arrays[f"fill.{v}"]).double()
        assert torch.all((f - g).abs() <= TOL * g.abs()), (v, f, g)
    l0 = want[0, 3].abs()
    inc = torch.from_numpy(arrays["increase"]).double()
    assert torch.all((imp["increase"] - inc).abs() <= TOL * (want[1:, 3].abs() + l0))
    sens = wo.feature_sensitivity(params64(arrays, meta), batch_of(arrays), cfg_of(meta),
                                  state_starts=meta["state_starts"],
                                  perm=torch.from_numpy(arrays["perm"]))
    err = np.abs(sens.numpy() - arrays["sensitivity"])
    assert np.all(err <= sensitivity_tol(arrays, meta)), (sens, arrays["sensitivity"])


def test_enum_fill_takes_the_first_column_at_the_lower_median():
    """The continuous golden's enum groups: a tie at the lower median, and a 2-column action
    group whose lower median (40, column 1) is not its upper one (59, column 0)."""
    arrays, meta = load("wm_eval_continuous_groups")
    # variants: original, action [0, 1), action [1, 3), state [0,1) [1,5) [5,6) [6,9) [9,10)
    np.testing.assert_array_equal(arrays["fill.2"], [0, 1])
    np.testing.assert_array_equal(arrays["fill.4"], [1, 0, 0, 0])  # counts 20 49 10 20
    np.testing.assert_array_equal(arrays["fill.6"], [0, 1, 0])     # counts 15 40 44
    f = torch.tensor([[1, 0], [0, 1], [1, 0]], dtype=torch.float64)
    np.testing.assert_array_equal(wo.fill_value(f).numpy(), [0, 1])


@pytest.mark.skipif(not reference_available(), reason="reference checkout not present")
def test_golden_regenerates_from_reference(tmp_path, monkeypatch):
    """The committed goldens are what the unmodified reference evaluators produce today."""
    from oracle import make_golden, make_world_model_eval_golden

    monkeypatch.setattr(make_golden, "GOLDEN", str(tmp_path))
    make_world_model_eval_golden.main({"wm_eval_continuous_groups", "wm_eval_fit_last_terminal"})
    for name in ("wm_eval_continuous_groups", "wm_eval_fit_last_terminal"):
        new = np.load(tmp_path / f"{name}.npz")
        old, _ = load(name)
        for k, v in old.items():
            np.testing.assert_array_equal(new[k], v, err_msg=f"{name}:{k}")


# ---------------------------------------------------------------------------------------------
# grouping and the variant table
# ---------------------------------------------------------------------------------------------
def test_feature_groups():
    assert feature_groups([0, 1, 5, 6, 9], 10, 5, "s") == [(0, 1), (1, 5), (5, 6), (6, 9), (9, 10)]
    assert feature_groups([0], 3, 1, "s") == [(0, 3)]


@pytest.mark.parametrize("starts,dim,num", [
    ([1, 2], 4, 2),      # does not start at 0
    ([0, 2, 2], 4, 3),   # not strictly increasing
    ([0, 3, 1], 4, 3),
    ([0, 4], 4, 2),      # a feature past the dimension
    ([0, 5], 4, 2),
    ([0, 1], 4, 3),      # fewer starts than features
    ([], 4, 0),
])
def test_malformed_feature_boundaries_are_refused(starts, dim, num):
    with pytest.raises(ValueError, match="feature"):
        feature_groups(starts, dim, num, "state features")


def test_variant_table_discrete():
    rows, n_eye, groups = importance_variants(True, 2, 4, None, [(0, 1), (1, 2), (2, 3), (3, 4)])
    assert n_eye == 4
    assert rows == [(0, 0, 0), (0, 2, 0), (0, 2, 2), (2, 3, 6), (3, 4, 7), (4, 5, 8), (5, 6, 9)]
    assert groups == [(2, 3), (3, 4), (4, 5), (5, 6)]


def test_variant_table_continuous():
    rows, n_eye, groups = importance_variants(False, 3, 10, [(0, 1), (1, 3)],
                                              [(0, 1), (1, 5), (5, 6), (6, 9), (9, 10)])
    assert n_eye == 0
    assert rows == [(0, 0, 0), (0, 1, 0), (1, 3, 1), (3, 4, 3), (4, 8, 4), (8, 9, 8),
                    (9, 12, 9), (12, 13, 12)]
    assert groups == [(0, 1), (1, 3), (3, 4), (4, 8), (8, 9), (9, 12), (12, 13)]


def test_variant_table_replays_the_oracle_on_the_materialised_batch():
    """Applying the table to x = cat(action, state) with the oracle's fills gives the same
    perturbed inputs as the oracle's per-feature clones."""
    arrays, meta = load("wm_eval_continuous_groups")
    A, S = meta["A"], meta["S"]
    b = batch_of(arrays)
    ev = FeatureImportanceEvaluator(None, False, len(meta["state_starts"]),
                                    len(meta["action_starts"]), meta["action_starts"],
                                    meta["state_starts"])
    rows, n_eye, groups = ev.variants(A, S)
    x = torch.cat([b["action"], b["state"]], dim=-1).reshape(-1, A + S)
    fill = torch.zeros(n_eye + A + S, dtype=torch.float64)
    for g0, g1 in groups:
        fill[n_eye + g0:n_eye + g1] = wo.fill_value(x[:, g0:g1])
    imp = importance_of(arrays, meta)
    for v, (c0, c1, off) in enumerate(rows[1:], start=1):
        np.testing.assert_array_equal(fill[off:off + c1 - c0].numpy(), imp["fills"][v].numpy())


# ---------------------------------------------------------------------------------------------
# constructors and refusals without CUDA
# ---------------------------------------------------------------------------------------------
def _trainer(S=4, A=2):
    torch.manual_seed(0)
    return MDNRNNTrainer(MemoryNetwork(S, A, 8, 1, 2), MDNRNNTrainerParameters(action_dim=A))


def _cpu_batch(T=2, B=3, S=4, A=2):
    z = lambda *s: torch.zeros(*s)  # noqa: E731
    return rlt.MemoryNetworkInput(state=rlt.FeatureData(z(T, B, S)),
                                  next_state=rlt.FeatureData(z(T, B, S)),
                                  action=rlt.FeatureData(z(T, B, A)), reward=z(T, B),
                                  not_terminal=z(T, B), time_diff=None, step=None)


def test_constructors_keep_the_reference_fields():
    tr = _trainer()
    le = LossEvaluator(tr, state_dim=4)
    assert (le.trainer, le.state_dim) == (tr, 4)
    fi = FeatureImportanceEvaluator(tr, discrete_action=True, state_feature_num=4,
                                    action_feature_num=2,
                                    sorted_action_feature_start_indices=[0, 1],
                                    sorted_state_feature_start_indices=[0, 1, 2, 3])
    assert (fi.trainer, fi.discrete_action, fi.state_feature_num, fi.action_feature_num) == (
        tr, True, 4, 2)
    assert fi.sorted_action_feature_start_indices == [0, 1]
    assert fi.sorted_state_feature_start_indices == [0, 1, 2, 3]
    fs = FeatureSensitivityEvaluator(tr, state_feature_num=4,
                                     sorted_state_feature_start_indices=[0, 1, 2, 3])
    assert (fs.trainer, fs.state_feature_num, fs.sorted_state_feature_start_indices) == (
        tr, 4, [0, 1, 2, 3])


def test_cpu_tensors_are_refused():
    tr = _trainer()
    b = _cpu_batch()
    for ev in (LossEvaluator(tr, 4),
               FeatureImportanceEvaluator(tr, True, 4, 2, [0, 1], [0, 1, 2, 3]),
               FeatureSensitivityEvaluator(tr, 4, [0, 1, 2, 3])):
        with pytest.raises(_lib.Rb200Error, match="CUDA"):
            ev.evaluate(b)


def test_non_sequence_inputs_are_refused(monkeypatch):
    """A [B, dim] state is refused before any device work (the CUDA check is bypassed)."""
    from reagent_b200.evaluation import world_model_evaluator as wme

    class FakeCuda(torch.Tensor):
        is_cuda = True

    tr = _trainer()
    b = _cpu_batch()
    b = rlt.MemoryNetworkInput(state=rlt.FeatureData(torch.zeros(3, 4).as_subclass(FakeCuda)),
                               next_state=b.next_state, action=b.action, reward=b.reward,
                               not_terminal=b.not_terminal, time_diff=None, step=None)
    with pytest.raises(ValueError, match=r"\[T, B, dim\]"):
        LossEvaluator(tr, 4).evaluate(b)
    with pytest.raises(TypeError, match="MemoryNetworkInput"):
        LossEvaluator(tr, 4).evaluate(object())


def test_discrete_importance_needs_one_feature_per_action():
    ev = FeatureImportanceEvaluator(None, True, 4, 3, [0, 1, 2], [0, 1, 2, 3])
    with pytest.raises(AssertionError):
        ev.variants(2, 4)


def test_eval_limits_are_in_the_header():
    assert _lib.MDNRNN_EVAL_MAX_VARIANTS == 1 + _lib.MDNRNN_MAX_INPUT == 257
    e = _lib.MdnrnnEvalArgsT()
    assert len(e.col_begin) == len(e.col_end) == len(e.fill_off) == 257
