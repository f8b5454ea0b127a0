"""The cross-entropy-method planner on the host: the fp64 oracle against the reference's
goldens, the parameters, the refusals and the limits."""
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cem_oracle  # noqa: E402
from oracle.ref_harness import reference_available  # noqa: E402
from tests.cem_cases import (CASES, assert_plans_match, cfg_of, fp64, noise_of,  # noqa: E402
                             planner_of, seeded_params, seeded_world_models)
from tests.golden_util import load  # noqa: E402

from reagent_b200 import _lib  # noqa: E402
from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import CEMTrainerParameters, MDNRNNTrainerParameters  # noqa: E402
from reagent_b200.models import CEMPlannerNetwork, MemoryNetwork  # noqa: E402


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_golden(name):
    arrays, meta = load(name)
    P = seeded_params(arrays, meta)
    cfg = cfg_of(meta)
    res = cem_oracle.plan(fp64(P), cfg, arrays["state"].astype(np.float64), noise_of(arrays))
    assert res["violations"] == []
    assert res["n_iters"] == meta["n_iters"]
    assert_plans_match(res, arrays, meta["discrete"], name)


@pytest.mark.parametrize("name", CASES)
def test_seeded_world_models_match_golden(name):
    """The discarded first build, then num_world_models MemoryNetworks, as the manager builds."""
    arrays, meta = load(name)
    seeded_world_models(arrays, meta)


@pytest.mark.skipif(not reference_available(), reason="reference checkout not present")
def test_golden_regenerates_from_reference(tmp_path, monkeypatch):
    """The committed golden is what the unmodified reference produces today."""
    from oracle import make_cem_golden, make_golden

    monkeypatch.setattr(make_golden, "GOLDEN", str(tmp_path))
    make_cem_golden.main({"cem_odd"})
    new = np.load(tmp_path / "cem_odd.npz")
    old, _ = load("cem_odd")
    for k, v in old.items():
        np.testing.assert_array_equal(new[k], v, err_msg=k)


@pytest.mark.skipif(not reference_available(), reason="reference checkout not present")
def test_parameters_match_reference():
    from oracle.ref_harness import ref

    theirs = ref("reagent.core.parameters").CEMTrainerParameters()
    ours = CEMTrainerParameters()
    for f in dataclasses.fields(ours):
        a, b = getattr(ours, f.name), getattr(theirs, f.name)
        if dataclasses.is_dataclass(a):
            for g in dataclasses.fields(a):
                assert getattr(a, g.name) == getattr(b, g.name), (f.name, g.name)
        else:
            assert a == b, f.name


def test_parameter_defaults_and_manager():
    from reagent_b200.model_managers import CrossEntropyMethod

    p = CEMTrainerParameters()
    assert (p.plan_horizon_length, p.num_world_models, p.cem_population_size,
            p.cem_num_iterations, p.ensemble_population_size, p.num_elites) == (0,) * 6
    assert (p.alpha, p.epsilon) == (0.25, 0.001)
    assert p.mdnrnn == MDNRNNTrainerParameters() and p.rl.gamma == 0.9
    m = CrossEntropyMethod()
    assert m.trainer_param == p
    with pytest.raises(RuntimeError):
        m.build_trainer({}, use_gpu=False)


def _planner(nets=None, **kw):
    nets = nets or [MemoryNetwork(4, 2, 8, 2, 1)]
    args = dict(mem_net_list=nets, cem_num_iterations=2, cem_population_size=20,
                ensemble_population_size=1, num_elites=5, plan_horizon_length=3, state_dim=4,
                action_dim=2, discrete_action=True, terminal_effective=True, gamma=1.0)
    args.update(kw)
    return CEMPlannerNetwork(**args)


def test_refusals():
    with pytest.raises(ValueError, match="ensemble_population_size must be 1"):
        _planner(ensemble_population_size=2)
    with pytest.raises(ValueError, match="one shape"):
        _planner([MemoryNetwork(4, 2, 8, 2, 1), MemoryNetwork(4, 2, 9, 2, 1)])
    with pytest.raises(ValueError, match="state_dim"):
        _planner(state_dim=5)
    with pytest.raises(NotImplementedError):
        _planner([torch.nn.Linear(2, 2)])
    pl = _planner()
    with pytest.raises(_lib.Rb200Error, match="CUDA only"):
        pl(rlt.FeatureData(torch.zeros(1, 4)))
    with pytest.raises(_lib.Rb200Error, match="CUDA only"):
        pl.plan(torch.zeros(1, 4))


# (S, A, hidden, layers, gaussians, population, models, horizon, num_elites)
AT_LIMIT = [(4, 2, 8, 2, 1, 1024, 1, 3, 1), (4, 2, 8, 2, 1, 10, 8, 3, 10),
            (4, 2, 8, 2, 1, 10, 1, 2048, 10), (200, 56, 128, 4, 2, 10, 1, 16, 1)]
PAST_LIMIT = [(4, 2, 8, 2, 1, 1025, 1, 3, 1), (4, 2, 8, 2, 1, 10, 9, 3, 5),
              (4, 2, 8, 2, 1, 10, 1, 2049, 5), (4, 2, 8, 2, 1, 10, 1, 3, 11),
              (4, 2, 8, 2, 1, 10, 1, 3, 0), (4, 2, 8, 2, 1, 10, 1, 0, 5),
              (4, 2, 129, 2, 1, 10, 1, 3, 5), (200, 57, 8, 1, 1, 10, 1, 3, 5)]


@pytest.mark.parametrize("shape", AT_LIMIT)
def test_shape_at_limit_accepted(shape):
    assert _lib.lib().rb200_cem_check_shape(*shape) == 0


@pytest.mark.parametrize("shape", PAST_LIMIT)
def test_shape_past_limit_refused(shape):
    assert _lib.lib().rb200_cem_check_shape(*shape) == -1
    S, A, H, L, G, P, K, hor, E = shape
    if H > 128:
        nets = [MemoryNetwork(S, A, H, L, G)]
    else:
        nets = [MemoryNetwork(S, A, H, L, G) for _ in range(min(K, 9))]
    with pytest.raises(_lib.Rb200Error, match="unsupported shape"):
        _planner(nets, cem_population_size=P, plan_horizon_length=hor, num_elites=E,
                 state_dim=S, action_dim=A)
