"""MDN-RNN on the host: the fp64 oracle against the reference's goldens, the API surface
(parameters, state_dict, seeded initial weights, optimizers) and the refusals."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mdnrnn_oracle as mo  # noqa: E402
from oracle.ref_harness import reference_available  # noqa: E402
from tests.golden_util import grad_close, load, rel_err  # noqa: E402

from reagent_b200 import _lib  # noqa: E402
from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import MDNRNNTrainerParameters  # noqa: E402
from reagent_b200.models import MemoryNetwork  # noqa: E402
from reagent_b200.optimizer import FusedAdam  # noqa: E402
from reagent_b200.training import MDNRNNTrainer  # noqa: E402

CASES = ["mdnrnn_cartpole_features", "mdnrnn_cem_cartpole", "mdnrnn_defaults_seq",
         "mdnrnn_fit_last_odd"]


def _initial(arrays, meta, requires_grad=False):
    """The case's seeded initial parameters in fp64, after checking their fp32 bits against the
    golden's digests."""
    P = mo.initial_params(meta["seed"], meta["S"], meta["A"], meta["H"], meta["L"], meta["G"])
    for i, p in enumerate(P):
        np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{i}.sha256"], err_msg=f"p0.{i}")
    return [p.double().requires_grad_(requires_grad) for p in P]


def _batch(arrays, it, dtype=torch.float64):
    return {k: torch.from_numpy(arrays[f"batch{it}.{k}"]).to(dtype)
            for k in ("state", "action", "next_state", "reward", "not_terminal")}


def _cfg(meta):
    return dict(L=meta["L"], G=meta["G"], next_state_weight=meta["next_state_weight"],
                not_terminal_weight=meta["not_terminal_weight"],
                reward_weight=meta["reward_weight"],
                fit_only_one_next_step=meta["fit_only_one_next_step"])


def _loss_kw(meta):
    return dict(next_state_weight=meta["next_state_weight"],
                not_terminal_weight=meta["not_terminal_weight"],
                reward_weight=meta["reward_weight"],
                fit_only_one_next_step=meta["fit_only_one_next_step"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_golden(name):
    arrays, meta = load(name)
    P = _initial(arrays, meta)
    b = _batch(arrays, 0)
    out = mo.forward(P, b["state"], b["action"], meta["L"], meta["G"])
    n = arrays["out.mus"].shape[1]
    for f in mo_fields():
        assert rel_err(out[f][:, :n], arrays[f"out.{f}"]) < 1e-5, f
    for key, sd in (("loss_sd", meta["S"]), ("loss", None)):
        ls = mo.losses(out, b["next_state"], b["reward"], b["not_terminal"], state_dim=sd,
                       **_loss_kw(meta))
        for k in mo.LOSS_KEYS:
            assert rel_err(ls[k], arrays[f"{key}.{k}"]) < 1e-5, (key, k)
    P = _initial(arrays, meta, requires_grad=True)
    opt = torch.optim.Adam(P, lr=meta["lr"])
    for it in range(meta["n_updates"]):
        ls, grads = mo.update(P, opt, _batch(arrays, it), _cfg(meta))
        assert rel_err(ls["loss"], arrays["losses"][it]) < 1e-5
        if it == 0:
            for i, g in enumerate(grads):
                grad_close(mo.sample(g), arrays[f"grad.{i}"], f"grad.{i}", l2_tol=1e-5,
                           max_tol=1e-4)
        for i, p in enumerate(P):
            d = (mo.sample(p.detach()) - torch.from_numpy(arrays[f"p{it + 1}.{i}"]).double()).abs()
            # Adam steps of at most lr each; elements with a near-zero gradient may differ by
            # a step's sign, everything else agrees far below one step
            assert float(d.max()) <= 2.0 * (it + 1) * meta["lr"] * 1.01, (it, i)
            assert float(d.median()) < 0.02 * meta["lr"], (it, i)


def mo_fields():
    return ("mus", "sigmas", "logpi", "reward", "not_terminal", "last_step_lstm_hidden",
            "last_step_lstm_cell", "all_steps_lstm_hidden")


@pytest.mark.skipif(not reference_available(), reason="reference checkout not present")
def test_golden_regenerates_from_reference(tmp_path, monkeypatch):
    """The committed golden is what the unmodified reference produces today."""
    from oracle import make_golden, make_mdnrnn_golden

    monkeypatch.setattr(make_golden, "GOLDEN", str(tmp_path))
    make_mdnrnn_golden.main({"mdnrnn_fit_last_odd", "memory_input_maker"})
    for name in ("mdnrnn_fit_last_odd", "memory_input_maker"):
        new = np.load(tmp_path / f"{name}.npz")
        old, _ = load(name)
        for k, v in old.items():
            np.testing.assert_array_equal(new[k], v, err_msg=f"{name}:{k}")


@pytest.mark.skipif(not reference_available(), reason="reference checkout not present")
def test_parameters_match_reference():
    import dataclasses

    from oracle.ref_harness import ref

    theirs = ref("reagent.core.parameters").MDNRNNTrainerParameters()
    ours = MDNRNNTrainerParameters()
    for f in dataclasses.fields(ours):
        assert getattr(ours, f.name) == getattr(theirs, f.name), f.name


def test_parameter_defaults_and_manager():
    from reagent_b200.model_managers import WorldModel

    p = MDNRNNTrainerParameters()
    assert (p.hidden_size, p.num_hidden_layers, p.learning_rate, p.num_gaussians) == (64, 2, 1e-3, 5)
    assert (p.reward_loss_weight, p.next_state_loss_weight, p.not_terminal_loss_weight) == (1.0,) * 3
    assert (p.fit_only_one_next_step, p.action_dim, p.action_names, p.multi_steps) == (False, 2, None, 1)
    m = WorldModel()
    assert m.trainer_param == p and m.reward_boost is None
    with pytest.raises(RuntimeError):
        m.build_trainer({}, use_gpu=False)


@pytest.mark.parametrize("name", CASES)
def test_seeded_initial_weights_and_keys(name):
    arrays, meta = load(name)
    torch.manual_seed(meta["seed"])
    net = MemoryNetwork(meta["S"], meta["A"], meta["H"], meta["L"], meta["G"])
    keys = list(net.state_dict().keys())
    want = []
    for l in range(meta["L"]):
        want += [f"mdnrnn.rnn.{w}_l{l}" for w in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    assert keys == want + ["mdnrnn.gmm_linear.weight", "mdnrnn.gmm_linear.bias"]
    params = list(net.mdnrnn.parameters())
    flat = net.arena.flat
    for i, p in enumerate(params):
        np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{i}.sha256"], err_msg=f"p0.{i}")
        # every parameter is a view of the one arena, in parameters() order
        assert p.data.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
        assert (p.data_ptr() - flat.data_ptr()) // 4 == net.arena.offsets[i]


def test_optimizers_and_yields():
    net = MemoryNetwork(4, 2, 8, 2, 1)
    tr = MDNRNNTrainer(net, MDNRNNTrainerParameters(learning_rate=3e-3))
    opts = tr.configure_optimizers()
    assert len(opts) == 1 and type(opts[0]) is FusedAdam
    g = opts[0].param_groups[0]
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"]) == (3e-3, (0.9, 0.999), 1e-8, 0.0)
    assert opts[0].arena is net.arena
    assert len(tr.optimizers()) == 1 and tr.optimizers()[0] is tr.optimizers()[0]


def _cpu_batch(T=2, B=3, S=4, A=2):
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(torch.randn(T, B, S)), next_state=rlt.FeatureData(torch.randn(T, B, S)),
        action=rlt.FeatureData(torch.randn(T, B, A)), reward=torch.randn(T, B),
        not_terminal=torch.ones(T, B), time_diff=None, step=None)


def test_refusals():
    net = MemoryNetwork(4, 2, 8, 2, 1)
    b = _cpu_batch()
    with pytest.raises(NotImplementedError):
        net.mdnrnn(b.action.float_features, b.state.float_features,
                   hidden=(torch.zeros(2, 3, 8), torch.zeros(2, 3, 8)))
    with pytest.raises(_lib.Rb200Error, match="CUDA only"):
        net(b.state, b.action)
    tr = MDNRNNTrainer(net, MDNRNNTrainerParameters())
    with pytest.raises(_lib.Rb200Error, match="CUDA only"):
        next(tr.train_step_gen(b, 0))
    with pytest.raises(_lib.Rb200Error, match="CUDA only"):
        tr.train_batch(b)
    with pytest.raises(NotImplementedError):
        MDNRNNTrainer(torch.nn.Linear(2, 2), MDNRNNTrainerParameters())


# (state_dim, action_dim, hidden, layers, gaussians) at each limit, and one past it
AT_LIMIT = [(4, 2, 128, 2, 1), (4, 2, 64, 4, 1), (4, 2, 8, 2, 32), (200, 56, 8, 1, 1),
            (255, 1, 8, 1, 2)]
PAST_LIMIT = [(4, 2, 129, 2, 1), (4, 2, 64, 5, 1), (2, 2, 8, 2, 33), (200, 57, 8, 1, 1),
              (255, 1, 8, 1, 3), (4, 2, 0, 2, 1)]


@pytest.mark.parametrize("shape", AT_LIMIT)
def test_shape_at_limit_accepted(shape):
    assert _lib.lib().rb200_mdnrnn_check_shape(*shape) == 0


@pytest.mark.parametrize("shape", PAST_LIMIT)
def test_shape_past_limit_refused(shape):
    net = MemoryNetwork(*shape) if shape[2] > 0 else None
    assert _lib.lib().rb200_mdnrnn_check_shape(*shape) == -1
    if net is not None:
        T, B = 1, 2
        # refused before the device check: the batch is on the CPU
        with pytest.raises(_lib.Rb200Error, match="unsupported shape"):
            net(rlt.FeatureData(torch.zeros(T, B, shape[0])), rlt.FeatureData(torch.zeros(T, B, shape[1])))


@pytest.mark.parametrize("kind,num_actions", [("discrete", 3), ("continuous", None)])
def test_input_maker_matches_reference(kind, num_actions):
    """MemoryNetworkInputMaker on the reference ReplayBuffer's samples (layout only)."""
    from types import SimpleNamespace

    from reagent_b200.gym.preprocessors.trainer_preprocessor import MemoryNetworkInputMaker

    arrays, _ = load("memory_input_maker")
    s = SimpleNamespace(**{f: torch.from_numpy(arrays[f"{kind}.sample.{f}"])
                           for f in ("state", "action", "reward", "next_state", "terminal")})
    out = MemoryNetworkInputMaker(num_actions)(s)
    got = dict(state=out.state.float_features, action=out.action.float_features,
               next_state=out.next_state.float_features, reward=out.reward,
               not_terminal=out.not_terminal)
    for f, v in got.items():
        np.testing.assert_array_equal(v.numpy(), arrays[f"{kind}.out.{f}"], err_msg=f)
    assert len(out) == s.state.shape[0]
