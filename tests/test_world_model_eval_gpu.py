"""World-model evaluators on the H100: the reference's goldens, each variant bit-identical to
MDNRNNTrainer.get_loss / MemoryNetwork.forward on the materialised batch, the fp64 oracle over
batch and sequence sizes and at the largest variant count, repeatability, no effect on
training, and the reference's CartPole assertion end to end."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mdnrnn_oracle as mo  # noqa: E402
from oracle import world_model_eval_oracle as wo  # noqa: E402
from tests.golden_util import load  # noqa: E402
from tests.world_model_eval_cases import CASES, TOL, sensitivity_tol  # noqa: E402

from reagent_b200 import _lib  # noqa: E402
from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import (MDNRNNTrainerParameters, NormalizationData,  # noqa: E402
                                          NormalizationKey, NormalizationParameters)
from reagent_b200.evaluation import (FeatureImportanceEvaluator,  # noqa: E402
                                     FeatureSensitivityEvaluator, LossEvaluator)
from reagent_b200.models import MemoryNetwork  # noqa: E402
from reagent_b200.training import MDNRNNTrainer  # noqa: E402

pytestmark = pytest.mark.gpu


def _params(meta):
    return MDNRNNTrainerParameters(
        hidden_size=meta["H"], num_hidden_layers=meta["L"], num_gaussians=meta["G"],
        reward_loss_weight=meta["reward_weight"], next_state_loss_weight=meta["next_state_weight"],
        not_terminal_loss_weight=meta["not_terminal_weight"],
        fit_only_one_next_step=meta["fit_only_one_next_step"], action_dim=meta["A"])


def _golden_trainer(arrays, meta):
    torch.manual_seed(meta["seed"])
    net = MemoryNetwork(meta["S"], meta["A"], meta["H"], meta["L"], meta["G"]).cuda()
    for i, p in enumerate(net.mdnrnn.parameters()):
        np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{i}.sha256"], err_msg=f"p0.{i}")
    return MDNRNNTrainer(net, _params(meta))


def _input(d):
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(d["state"]), next_state=rlt.FeatureData(d["next_state"]),
        action=rlt.FeatureData(d["action"]), reward=d["reward"], not_terminal=d["not_terminal"],
        time_diff=None, step=None)


def _golden_batch(arrays):
    return _input({k: torch.from_numpy(arrays[f"batch.{k}"]).cuda()
                   for k in ("state", "action", "next_state", "reward", "not_terminal")})


def _evaluators(tr, meta):
    imp = FeatureImportanceEvaluator(
        tr, discrete_action=meta["discrete"], state_feature_num=len(meta["state_starts"]),
        action_feature_num=meta["action_feature_num"],
        sorted_action_feature_start_indices=meta["action_starts"],
        sorted_state_feature_start_indices=meta["state_starts"])
    sens = FeatureSensitivityEvaluator(tr, state_feature_num=len(meta["state_starts"]),
                                       sorted_state_feature_start_indices=meta["state_starts"])
    return imp, sens


def _variant_fills(imp, A, S):
    rows, _, _ = imp.variants(A, S)
    fill = imp.fill_values().cpu()
    return rows, [fill[off:off + c1 - c0] for c0, c1, off in rows]


def _materialise(batch, c0, c1, value, A):
    """The batch with columns [c0, c1) of x = cat(action, state) set to `value` everywhere."""
    x = torch.cat([batch.action.float_features, batch.state.float_features], dim=-1).clone()
    x[:, :, c0:c1] = value.to(x.device)
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(x[:, :, A:].contiguous()), next_state=batch.next_state,
        action=rlt.FeatureData(x[:, :, :A].contiguous()), reward=batch.reward,
        not_terminal=batch.not_terminal, time_diff=None, step=None)


@pytest.mark.parametrize("name", CASES)
def test_golden(name):
    arrays, meta = load(name)
    tr = _golden_trainer(arrays, meta)
    imp, sens = _evaluators(tr, meta)
    batch = _golden_batch(arrays)
    inc = imp.evaluate(batch)["feature_loss_increase"]
    assert inc.dtype == np.float32 and inc.shape == arrays["increase"].shape
    losses = imp._bufs.loss.cpu().double().numpy()
    want = arrays["losses"]
    assert np.all(np.abs(losses - want) <= TOL * np.abs(want)), (losses, want)
    assert np.all(np.abs(inc - arrays["increase"]) <= TOL * (np.abs(want[1:, 3]) + abs(want[0, 3])))
    _, fills = _variant_fills(imp, meta["A"], meta["S"])
    for v in range(1, len(fills)):
        g = arrays[f"fill.{v}"]
        assert np.all(np.abs(fills[v].numpy() - g) <= TOL * np.abs(g)), (v, fills[v], g)

    B = meta["B"]
    torch.manual_seed(meta["perm_seed"])
    assert torch.equal(torch.randperm(B), torch.from_numpy(arrays["perm"]))
    torch.manual_seed(meta["perm_seed"])
    s = sens.evaluate(batch)["feature_sensitivity"]
    assert s.dtype == np.float32 and s.shape == arrays["sensitivity"].shape
    assert np.all(np.abs(s - arrays["sensitivity"]) <= sensitivity_tol(arrays, meta))
    s2 = sens.evaluate(batch, perm=torch.from_numpy(arrays["perm"]))["feature_sensitivity"]
    np.testing.assert_array_equal(s, s2)

    lo = LossEvaluator(tr, meta["S"]).evaluate(batch)
    assert list(lo) == ["loss", "gmm", "bce", "mse"]
    assert all(isinstance(v, float) for v in lo.values())
    np.testing.assert_array_equal([lo[k] for k in ("gmm", "bce", "mse", "loss")],
                                  imp._bufs.loss[0].cpu().numpy())


@pytest.mark.parametrize("name", CASES)
def test_variants_are_bit_identical_to_get_loss_and_forward(name):
    arrays, meta = load(name)
    tr = _golden_trainer(arrays, meta)
    imp, sens = _evaluators(tr, meta)
    batch = _golden_batch(arrays)
    A, S = meta["A"], meta["S"]
    imp.evaluate(batch)
    got = imp._bufs.loss.clone()
    rows, fills = _variant_fills(imp, A, S)
    for v, (c0, c1, _) in enumerate(rows):
        ls = tr.get_loss(_materialise(batch, c0, c1, fills[v], A), state_dim=S)
        want = torch.stack([ls[k] for k in ("gmm", "bce", "mse", "loss")])
        assert torch.equal(got[v], want), (v, got[v], want)

    perm = torch.from_numpy(arrays["perm"])
    sens.evaluate(batch, perm=perm)
    mus = sens.means()
    with torch.no_grad():
        m0 = tr.memory_network(batch.state, batch.action).mus.clone()
        m1 = tr.memory_network(batch.state, rlt.FeatureData(
            batch.action.float_features[:, perm.cuda(), :])).mus.clone()
    assert torch.equal(mus[0], m0)
    assert torch.equal(mus[1], m1)


def _random_case(T, B, S, A, H, L, G, discrete, seed, fit_last=False):
    torch.manual_seed(seed)
    net = MemoryNetwork(S, A, H, L, G)
    P64 = [p.detach().double().clone() for p in net.mdnrnn.parameters()]
    params = MDNRNNTrainerParameters(hidden_size=H, num_hidden_layers=L, num_gaussians=G,
                                     action_dim=A, fit_only_one_next_step=fit_last)
    tr = MDNRNNTrainer(net.cuda(), params)
    g = torch.Generator().manual_seed(seed + 1)
    if discrete:
        action = torch.nn.functional.one_hot(torch.randint(A, (T, B), generator=g), A).float()
    else:
        action = torch.rand(T, B, A, generator=g) * 2 - 1
    d = dict(state=torch.randn(T, B, S, generator=g), action=action,
             next_state=torch.randn(T, B, S, generator=g), reward=torch.randn(T, B, generator=g),
             not_terminal=(torch.rand(T, B, generator=g) > 0.1).float())
    cfg = dict(L=L, G=G, next_state_weight=1.0, not_terminal_weight=1.0, reward_weight=1.0,
               fit_only_one_next_step=fit_last)
    return tr, P64, d, cfg


def _check_against_oracle(tr, P64, d, cfg, discrete, a_starts, s_starts, rtol=2e-5):
    T, B, S = d["state"].shape
    A = d["action"].shape[2]
    batch = _input({k: v.cuda() for k, v in d.items()})
    imp = FeatureImportanceEvaluator(tr, discrete, len(s_starts),
                                     A if discrete else len(a_starts), a_starts, s_starts)
    inc = imp.evaluate(batch)["feature_loss_increase"]
    b64 = {k: v.double() for k, v in d.items()}
    ref = wo.feature_importance(P64, b64, cfg, discrete_action=discrete, action_starts=a_starts,
                                state_starts=s_starts)
    losses = imp._bufs.loss.cpu().double()
    assert torch.all((losses - ref["losses"]).abs() <= rtol * ref["losses"].abs()), (
        losses, ref["losses"])
    tol = rtol * (ref["losses"][1:, 3].abs() + ref["losses"][0, 3].abs())
    assert torch.all((torch.from_numpy(inc).double() - ref["increase"]).abs() <= tol)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(5))
    sens = FeatureSensitivityEvaluator(tr, len(s_starts), s_starts)
    s = sens.evaluate(batch, perm=perm)["feature_sensitivity"]
    want = wo.feature_sensitivity(P64, b64, cfg, state_starts=s_starts, perm=perm)
    m0 = mo.forward(P64, b64["state"], b64["action"], cfg["L"], cfg["G"])["mus"]
    m1 = mo.forward(P64, b64["state"], b64["action"][:, perm], cfg["L"], cfg["G"])["mus"]
    stol = torch.stack([(m0[..., a:b].abs() + m1[..., a:b].abs()).sum(dim=3).mean()
                        for a, b in wo.groups(s_starts, S)]) * rtol
    assert torch.all((torch.from_numpy(s).double() - want).abs() <= stol), (s, want)


@pytest.mark.parametrize("T", [1, 6, 16])
@pytest.mark.parametrize("B", [1, 15, 17, 6000])
def test_against_fp64_oracle(T, B):
    tr, P64, d, cfg = _random_case(T, B, S=4, A=2, H=64, L=2, G=5, discrete=True, seed=T * B)
    _check_against_oracle(tr, P64, d, cfg, True, [0, 1], [0, 1, 2, 3])


def test_against_fp64_oracle_continuous_fit_last():
    tr, P64, d, cfg = _random_case(5, 33, S=6, A=3, H=24, L=3, G=3, discrete=False, seed=9,
                                   fit_last=True)
    d["state"][:, :, 2:5] = torch.nn.functional.one_hot(
        torch.arange(5 * 33).reshape(5, 33) % 3, 3).float()
    _check_against_oracle(tr, P64, d, cfg, False, [0, 2], [0, 1, 2, 5])


def test_largest_variant_count():
    """A + S = 256 width-1 features: 257 variants, the most the limits allow."""
    A, S = 1, 255
    tr, P64, d, cfg = _random_case(2, 17, S=S, A=A, H=8, L=1, G=1, discrete=False, seed=11)
    _check_against_oracle(tr, P64, d, cfg, False, [0], list(range(S)))
    assert _lib.MDNRNN_EVAL_MAX_VARIANTS == 1 + A + S


def test_limits_refused_by_the_c_abi():
    """Each refused table comes with buffers sized for it, so a launch that got through would
    still stay inside its allocations; only the refusal is under test."""
    from reagent_b200.evaluation.world_model_evaluator import _EvalBuffers

    T, B, S, A = 1, 4, 4, 2
    tr, _, d, _ = _random_case(T, B, S=S, A=A, H=8, L=1, G=1, discrete=True, seed=1)
    batch = _input({k: v.cuda() for k, v in d.items()})
    ev = LossEvaluator(tr, S)
    state, action, targets = ev._inputs(batch)
    for variants, n_fill in (([(0, 0, 0)] * 8, A + S),            # V > 1 + A + S
                             ([(0, 0, 0), (5, 7, 0)], A + S + 1),  # past A + S
                             ([(0, 0, 0), (3, 2, 0)], A + S),      # reversed
                             ([(0, 0, 0), (0, 2, 0)], 1)):         # past the fill values
        ws = _EvalBuffers(T, B, len(variants), n_fill, 0, state.device)
        ws.fill = torch.zeros(A + S + 2, device=state.device)[:n_fill]  # fill_len = n_fill
        with pytest.raises(_lib.Rb200Error, match="rb200_mdnrnn_eval"):
            ev._launch(state, action, targets, variants, ws)
    mus0, mus1 = (torch.zeros(T * B, 1, S, device="cuda") for _ in range(2))
    out = torch.zeros(2, device="cuda")
    e = _lib.MdnrnnSensitivityArgsT()
    e.rows, e.state_dim, e.gaussians, e.num_groups = T * B, S, 1, 2
    e.group_begin[0], e.group_begin[1], e.group_begin[2] = 0, 3, 2  # not increasing
    e.mus0, e.mus1, e.out = mus0.data_ptr(), mus1.data_ptr(), out.data_ptr()
    assert _lib.lib().rb200_mdnrnn_sensitivity(e, _lib.cur_stream()) == _lib.E_INVALID
    torch.cuda.synchronize()
    assert torch.equal(out, torch.zeros(2, device="cuda"))


def test_one_host_synchronisation_per_evaluate():
    """Each evaluate synchronises once, for its read-back: the permutation goes up from pinned
    memory without waiting for the stream."""
    import warnings

    tr, _, d, _ = _random_case(3, 50, S=4, A=2, H=16, L=1, G=2, discrete=False, seed=4)
    batch = _input({k: v.cuda() for k, v in d.items()})
    evaluators = [LossEvaluator(tr, 4),
                  FeatureImportanceEvaluator(tr, False, 4, 2, [0, 1], [0, 1, 2, 3]),
                  FeatureSensitivityEvaluator(tr, 4, [0, 1, 2, 3])]
    for ev in evaluators:
        ev.evaluate(batch)  # buffers and module loads outside the count
    torch.cuda.synchronize()
    for ev in evaluators:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                ev.evaluate(batch)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs = [w for w in caught if "synchronizing cuda operation" in str(w.message).lower()]
        assert len(syncs) == 1, (type(ev).__name__, [str(w.message) for w in syncs])


def test_loss_evaluator_divides_gmm_by_its_own_state_dim():
    """LossEvaluator(trainer, state_dim) is get_loss(batch, state_dim): its state_dim, not the
    batch's, sets the gmm divisor state_dim + 2."""
    tr, _, d, _ = _random_case(2, 33, S=4, A=2, H=16, L=2, G=2, discrete=True, seed=6)
    batch = _input({k: v.cuda() for k, v in d.items()})
    for sd in (4, 7):
        got = LossEvaluator(tr, sd).evaluate(batch)
        want = {k: float(v) for k, v in tr.get_loss(batch, state_dim=sd).items()}
        assert got == {k: want[k] for k in ("loss", "gmm", "bce", "mse")}, (sd, got, want)


def test_repeatable_and_leaves_training_unchanged():
    def run(evaluate):
        tr, _, d, _ = _random_case(6, 100, S=4, A=2, H=32, L=2, G=3, discrete=True, seed=3)
        batch = _input({k: v.cuda() for k, v in d.items()})
        imp = FeatureImportanceEvaluator(tr, True, 4, 2, [0, 1], [0, 1, 2, 3])
        sens = FeatureSensitivityEvaluator(tr, 4, [0, 1, 2, 3])
        out = [tr.train_batch(batch).clone()]
        if evaluate:
            r1 = imp.evaluate(batch)["feature_loss_increase"]
            torch.manual_seed(0)
            s1 = sens.evaluate(batch)["feature_sensitivity"]
            l1 = LossEvaluator(tr, 4).evaluate(batch)
            r2 = imp.evaluate(batch)["feature_loss_increase"]
            torch.manual_seed(0)
            s2 = sens.evaluate(batch)["feature_sensitivity"]
            l2 = LossEvaluator(tr, 4).evaluate(batch)
            np.testing.assert_array_equal(r1, r2)
            np.testing.assert_array_equal(s1, s2)
            assert l1 == l2
            assert tr.memory_network.mdnrnn.training
        out.append(tr.train_batch(batch).clone())
        return out, [p.detach().clone() for p in tr.memory_network.mdnrnn.parameters()]

    (la, pa), (lb, pb) = run(True), run(False)
    for x, y in zip(la + pa, lb + pb):
        assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------
# reagent/gym/tests/test_world_model.py::test_mdnrnn, with CartPole simulated here
# ---------------------------------------------------------------------------------------------
class CartPole:
    """CartPole-v0 (Barto, Sutton & Anderson 1983, as published in gym): force +-10 N, Euler
    steps of 0.02 s, reward 1 per step, the episode ends when |x| > 2.4 or |theta| > 12
    degrees, or after 200 steps; a new episode starts uniform in [-0.05, 0.05]^4."""

    gravity, masscart, masspole, length, force_mag, tau = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
    theta_limit, x_limit, max_steps = 12 * 2 * math.pi / 360, 2.4, 200

    def __init__(self, rng):
        self.rng = rng
        self.reset()

    def reset(self):
        self.s = self.rng.uniform(-0.05, 0.05, 4)
        self.t = 0
        return self.s.copy()

    def step(self, action):
        x, x_dot, theta, theta_dot = self.s
        force = self.force_mag if action == 1 else -self.force_mag
        cos, sin = math.cos(theta), math.sin(theta)
        total_mass = self.masspole + self.masscart
        pml = self.masspole * self.length
        temp = (force + pml * theta_dot ** 2 * sin) / total_mass
        theta_acc = (self.gravity * sin - cos * temp) / (
            self.length * (4.0 / 3.0 - self.masspole * cos ** 2 / total_mass))
        x_acc = temp - pml * theta_acc * cos / total_mass
        x, x_dot = x + self.tau * x_dot, x_dot + self.tau * x_acc
        theta, theta_dot = theta + self.tau * theta_dot, theta_dot + self.tau * theta_acc
        self.s = np.array([x, x_dot, theta, theta_dot])
        self.t += 1
        done = bool(abs(x) > self.x_limit or abs(theta) > self.theta_limit
                    or self.t >= self.max_steps)
        return self.s.copy(), 1.0, done


def _fill(rb, env, n, rng):
    """`n` random-policy transitions (observation before the action), as fill_replay_buffer
    adds them."""
    obs, act, rew, term = [], [], [], []
    s = env.reset()
    for _ in range(n):
        a = int(rng.randint(2))
        s2, r, done = env.step(a)
        obs.append(s)
        act.append(a)
        rew.append(r)
        term.append(done)
        s = env.reset() if done else s2
    rb.add_batch(observation=np.array(obs, dtype=np.float32), action=np.array(act),
                 reward=np.array(rew, dtype=np.float32), terminal=np.array(term))


def test_cartpole_feature_importance_and_sensitivity():
    """configs/world_model/cartpole_features.yaml as written: 100 000 training transitions,
    6 000 test transitions, seq_len 1, batch 1024, 30 epochs; the top importance is state1 or
    state3 and the top sensitivity is state3."""
    from reagent_b200.gym.preprocessors.trainer_preprocessor import MemoryNetworkInputMaker
    from reagent_b200.model_managers import WorldModel
    from reagent_b200.replay_memory.circular_replay_buffer import ReplayBuffer

    n_train, n_test, seq_len, batch_size, epochs = 100000, 6000, 1, 1024, 30
    torch.manual_seed(0)
    rng = np.random.RandomState(0)
    env = CartPole(rng)
    manager = WorldModel(trainer_param=MDNRNNTrainerParameters(
        hidden_size=50, num_hidden_layers=2, learning_rate=0.001, not_terminal_loss_weight=1,
        next_state_loss_weight=1, reward_loss_weight=1, num_gaussians=1))
    norm = {NormalizationKey.STATE: NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS") for i in range(4)})}
    tr = manager.build_trainer(norm, use_gpu=True)
    maker = MemoryNetworkInputMaker(2)

    def prep(s):
        s = type(s)(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v)
                       for k, v in s._asdict().items()})
        return maker(s)

    test_rb = ReplayBuffer(replay_capacity=n_test, batch_size=batch_size, stack_size=seq_len,
                           return_everything_as_stack=True)
    _fill(test_rb, env, n_test, rng)
    train_rb = ReplayBuffer(replay_capacity=n_train, batch_size=batch_size, stack_size=seq_len,
                            return_everything_as_stack=True)
    _fill(train_rb, env, n_train, rng)
    for _ in range(epochs):
        for i in range(train_rb.size // batch_size):
            tr.train_batch(prep(train_rb.sample_transition_batch(batch_size=batch_size)), i)

    test_batch = prep(test_rb.sample_transition_batch(batch_size=test_rb.size))
    imp = FeatureImportanceEvaluator(tr, discrete_action=True, state_feature_num=4,
                                     action_feature_num=2,
                                     sorted_action_feature_start_indices=[0, 1],
                                     sorted_state_feature_start_indices=[0, 1, 2, 3])
    sens = FeatureSensitivityEvaluator(tr, state_feature_num=4,
                                       sorted_state_feature_start_indices=[0, 1, 2, 3])
    fi = imp.evaluate(test_batch)["feature_loss_increase"]
    fs = sens.evaluate(test_batch)["feature_sensitivity"]
    names = ["action0", "action1", "state0", "state1", "state2", "state3"]
    importance = dict(zip(names, fi.tolist()))
    sensitivity = dict(zip(names[2:], fs.tolist()))
    print("feature importance", importance, "\nfeature sensitivity", sensitivity)
    assert max(importance, key=importance.get) in ("state1", "state3"), importance
    assert max(sensitivity, key=sensitivity.get) == "state3", sensitivity
