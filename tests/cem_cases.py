"""What the CEM planner tests share: the golden cases, their oracle configuration, noise and
seeded world models, and one comparison of two plans."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cem_oracle  # noqa: E402
from oracle import mdnrnn_oracle as mo  # noqa: E402

CASES = ["cem_cartpole_offline", "cem_linear_dynamics_single", "cem_linear_dynamics_many",
         "cem_odd"]
TRAINER_CASES = ["cem_cartpole_offline", "cem_linear_dynamics_many"]
TOL = 1e-5


def cfg_of(meta):
    return dict(discrete=meta["discrete"], K=meta["K"], P=meta["P"], H=meta["H"], A=meta["A"],
                S=meta["S"], L=meta["layers"], G=meta["G"], iters=meta["iters"],
                num_elites=meta["num_elites"], gamma=meta["gamma"], alpha=meta["alpha"],
                epsilon=meta["epsilon"], terminal_effective=meta["not_terminal_weight"] > 0,
                lower=meta["lower"], upper=meta["upper"])


def noise_of(arrays):
    return {k[len("noise."):]: v for k, v in arrays.items() if k.startswith("noise.")}


def seeded_params(arrays, meta):
    """The case's seeded world models (fp32, parameters() order), checked bit for bit against
    the golden's digests."""
    P = cem_oracle.initial_params(meta["seed"], meta["K"], meta["S"], meta["A"], meta["hidden"],
                                  meta["layers"], meta["G"])
    for m, ps in enumerate(P):
        for i, p in enumerate(ps):
            np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{m}.{i}.sha256"],
                                          err_msg=f"p0.{m}.{i}")
    return P


def assert_plans_match(got, want, discrete, what=""):
    """Values at 1e-5 (relative to max(1, |value|)), the same iteration count and elite sets,
    mean / var at 1e-5, and the action: the discrete index exactly, the continuous one at
    1e-5."""
    gv, wv = np.asarray(got["values"], np.float64), np.asarray(want["values"], np.float64)
    assert gv.shape == wv.shape, (what, "iterations / population", gv.shape, wv.shape)
    err = np.abs(gv - wv) / np.maximum(1.0, np.abs(wv))
    assert err.max() <= TOL, (what, "values", float(err.max()))
    if discrete:
        assert int(got["action"]) == int(want["action"]), (what, "action")
        return
    for i, (a, b) in enumerate(zip(got["elites"], want["elites"])):
        assert set(np.asarray(a).tolist()) == set(np.asarray(b).tolist()), (what, "elites", i)
    for k in ("mean", "var"):
        g, w = np.asarray(got[k], np.float64), np.asarray(want[k], np.float64)
        assert g.shape == w.shape, (what, k)
        err = np.abs(g - w) / np.maximum(1.0, np.abs(w))
        assert err.max() <= TOL, (what, k, float(err.max()))
    ga, wa = np.asarray(got["action"], np.float64), np.asarray(want["action"], np.float64)
    assert np.abs(ga - wa).max() <= TOL, (what, "action", ga, wa)


def fp64(params):
    return [[p.double() for p in ps] for ps in params]


def seeded_world_models(arrays, meta):
    """MemoryNetworks built as CrossEntropyMethod.build_trainer builds them (one discarded
    first) under the case's seed, checked against the golden's digests."""
    from reagent_b200.models import MemoryNetwork

    torch.manual_seed(meta["seed"])
    args = (meta["S"], meta["A"], meta["hidden"], meta["layers"], meta["G"])
    MemoryNetwork(*args)
    nets = [MemoryNetwork(*args) for _ in range(meta["K"])]
    for m, net in enumerate(nets):
        for i, p in enumerate(net.mdnrnn.parameters()):
            np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{m}.{i}.sha256"],
                                          err_msg=f"p0.{m}.{i}")
    return nets


def planner_of(nets, meta):
    from reagent_b200.models import CEMPlannerNetwork

    cont = not meta["discrete"]
    return CEMPlannerNetwork(
        mem_net_list=nets, cem_num_iterations=meta["iters"], cem_population_size=meta["P"],
        ensemble_population_size=1, num_elites=meta["num_elites"], plan_horizon_length=meta["H"],
        state_dim=meta["S"], action_dim=meta["A"], discrete_action=meta["discrete"],
        terminal_effective=meta["not_terminal_weight"] > 0, gamma=meta["gamma"],
        alpha=meta["alpha"], epsilon=meta["epsilon"],
        action_upper_bounds=np.array(meta["upper"]) if cont else None,
        action_lower_bounds=np.array(meta["lower"]) if cont else None)
