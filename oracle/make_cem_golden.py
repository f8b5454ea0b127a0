"""Generate the cross-entropy-method golden vectors in tests/golden/ by running the UNMODIFIED
reference CEMPlannerNetwork (reagent/models/cem_planner.py) and CEMTrainer (reagent/training/
cem_trainer.py) through oracle/ref_harness.py.  Needs the reference checkout (build container
only); the files are committed.

    python oracle/make_cem_golden.py            # regenerate every case
    python oracle/make_cem_golden.py NAME ...   # only the named ones

The reference manager (model_managers/model_based/cross_entropy_method.py) imports pyspark, so
the networks are built here the way its build_trainer builds them: under torch.manual_seed, one
MemoryNetwork built and discarded, then num_world_models MemoryNetworks with their
MDNRNNTrainers.

The planner's samplers are replaced, inside the reference's cem_planner module only, by shims
that read recorded noise (oracle/cem_oracle.py layout) by (iteration, solution, step):
np.random.randint (world model), random.choices (discrete action sequences), stats.truncnorm
(continuous solutions), Categorical, Normal and Bernoulli, with the formulas of the fused
kernel.  The noise is first guarded with oracle.cem_oracle.guard_noise, so no decision lies
near a boundary.

A case holds
  p0.{m}.{i}.sha256     SHA-256 of world model m's seeded parameters (parameters() order),
                        rebuilt by oracle.cem_oracle.initial_params
  state                 the planning state [S]
  noise.{model_idx, step, action_idx | truncnorm}
  values [n, P]         every iteration's solution values (n iterations run)
  elites [n, E]         np.argsort(values)[-num_elites:] of each iteration (continuous)
  mean / var [n, H*A]   after each iteration's update (continuous)
  action                discrete: the index, with one_hot [A]; continuous: the fp64 action [A]
A trainer case also holds batch{t}.*, `losses` [updates, K] and p{t}.{m}.{i}: world model m's
parameters after update t on oracle.mdnrnn_oracle.sample's subsample (make_mdnrnn_golden.py).
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import cem_oracle  # noqa: E402
from oracle.make_golden import _np, _save  # noqa: E402
from oracle.mdnrnn_oracle import digest, sample  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402

N_UPDATES = 2
TRAIN_T, TRAIN_B = 1, 256


class _Shims:
    """The reference planner's random draws, read from recorded noise."""

    def __init__(self, noise, S, discrete):
        self.noise, self.S, self.discrete = noise, S, discrete
        self.it = 0 if discrete else -1
        self.sol = -1
        self.step = -1
        self.elites, self.var_after, self.new_mean = [], [], []

    # np.random.randint(0, num_world_models): one call per trajectory, in solution order
    def randint(self, low, high=None, size=None):
        assert size is None
        self.sol += 1
        self.step = -1
        return int(self.noise["model_idx"][self.it, self.sol])

    # random.choices(product(range(A), repeat=H), k=P)
    def choices(self, population, k):
        assert k == self.noise["action_idx"].shape[0]
        self.sol = -1
        return [tuple(int(a) for a in row) for row in self.noise["action_idx"]]

    # stats.truncnorm(-2, 2, loc=0, scale=1).rvs(size=[P, H * A]): one call per iteration
    def truncnorm(self, a, b, loc, scale):
        assert (a, b) == (-2, 2) and np.all(loc == 0) and np.all(scale == 1)
        shims = self

        def rvs(size):
            shims.it += 1
            shims.sol = -1
            z = shims.noise["truncnorm"][shims.it]
            assert list(z.shape) == list(size)
            return z.copy()

        return SimpleNamespace(rvs=rvs)

    def _nz(self):
        return self.noise["step"][self.it, self.sol, self.step]

    def categorical(self, probs):
        shims = self

        def sample():
            shims.step += 1
            p = probs.detach().numpy().astype(np.float32)
            tot = np.float32(0)
            for q in p:
                tot = np.float32(tot + q)
            thr = np.float32(np.float32(shims._nz()[0]) * tot)
            cum, k = np.float32(0), len(p) - 1
            for q, pq in enumerate(p):
                cum = np.float32(cum + pq)
                if thr < cum:
                    k = q
                    break
            return torch.tensor(k)

        return SimpleNamespace(sample=sample)

    def normal(self, loc, scale):
        def sample():
            z = torch.from_numpy(self._nz()[1:self.S + 1].copy())
            return loc + scale * z

        return SimpleNamespace(sample=sample)

    def bernoulli(self, p):
        def sample():
            u = torch.tensor(float(self._nz()[self.S + 1]), dtype=torch.float32)
            return (u < p).float()

        return SimpleNamespace(sample=sample)


class _NpProxy:
    """numpy for the reference planner module, with np.random.randint shimmed and the elites
    (np.argsort) and the updated variance (np.max) recorded."""

    def __init__(self, shims, num_elites):
        self._sh, self._E = shims, num_elites
        self.random = SimpleNamespace(randint=shims.randint)

    def __getattr__(self, k):
        return getattr(np, k)

    def argsort(self, a, *args, **kw):
        r = np.argsort(a, *args, **kw)
        self._sh.elites.append(r[-self._E:].copy())
        return r

    def mean(self, a, *args, **kw):
        r = np.mean(a, *args, **kw)
        self._sh.new_mean.append(r.copy())
        return r

    def max(self, a, *args, **kw):
        self._sh.var_after.append(np.array(a, copy=True))
        return np.max(a, *args, **kw)


def _run_reference_planner(planner, cp, noise, state, cfg):
    sh = _Shims(noise, cfg["S"], cfg["discrete"])
    saved = {k: getattr(cp, k) for k in ("np", "random", "stats", "Categorical", "Normal", "Bernoulli")}
    cp.np = _NpProxy(sh, cfg["num_elites"])
    cp.random = SimpleNamespace(choices=sh.choices)
    cp.stats = SimpleNamespace(truncnorm=sh.truncnorm)
    cp.Categorical, cp.Normal, cp.Bernoulli = sh.categorical, sh.normal, sh.bernoulli
    values, mean_in = [], []
    orig_acc, orig_cv = planner.acc_rewards_of_all_solutions, planner.constrained_variance

    def acc(st, sols):
        v = orig_acc(st, sols)
        values.append(np.array(v, copy=True))
        return v

    def cv(mean, var):
        mean_in.append(np.array(mean, copy=True))
        return orig_cv(mean, var)

    planner.acc_rewards_of_all_solutions, planner.constrained_variance = acc, cv
    rlt = ref("reagent.core.types")
    try:
        out = planner(rlt.FeatureData(float_features=torch.from_numpy(state)[None]))
    finally:
        for k, v in saved.items():
            setattr(cp, k, v)
        del planner.acc_rewards_of_all_solutions, planner.constrained_variance
    res = dict(values=np.array(values))
    if cfg["discrete"]:
        res.update(action=np.array(out[0], dtype=np.int64), one_hot=_np(out[1]).copy())
    else:
        al = planner.alpha
        res.update(elites=np.array(sh.elites, dtype=np.int64), var=np.array(sh.var_after),
                   mean=np.array([al * m + (1 - al) * nm for m, nm in zip(mean_in, sh.new_mean)]),
                   action=_np(out).copy())
    return res


def _check_against_oracle(res, orc, cfg):
    """The guarded fp64 oracle agrees with the reference before anything is written."""
    assert res["values"].shape == np.asarray(orc["values"]).shape
    np.testing.assert_allclose(res["values"], orc["values"], rtol=1e-5, atol=1e-5)
    if cfg["discrete"]:
        assert int(res["action"]) == orc["action"]
    else:
        for a, b in zip(res["elites"], orc["elites"]):
            assert set(a.tolist()) == set(b.tolist())
        np.testing.assert_allclose(res["mean"], orc["mean"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(res["action"], orc["action"], rtol=1e-5, atol=1e-7)


def case(name, *, discrete, K, S, A, H, P, iters, E, gamma, hidden, layers, G, nt_weight,
         seed, trainer=False, lower=None, upper=None, alpha=0.25, epsilon=0.001):
    params_mod = ref("reagent.core.parameters")
    wm = ref("reagent.models.world_model")
    cp = ref("reagent.models.cem_planner")
    trainer_mod = ref("reagent.training.world_model.mdnrnn_trainer")
    cem_trainer_mod = ref("reagent.training.cem_trainer")
    rlt = ref("reagent.core.types")
    mdn = params_mod.MDNRNNTrainerParameters(hidden_size=hidden, num_hidden_layers=layers,
                                             num_gaussians=G, action_dim=A,
                                             not_terminal_loss_weight=nt_weight)
    cem = params_mod.CEMTrainerParameters(
        plan_horizon_length=H, num_world_models=K, cem_population_size=P,
        cem_num_iterations=iters, ensemble_population_size=1, num_elites=E, mdnrnn=mdn,
        rl=params_mod.RLParameters(gamma=gamma), alpha=alpha, epsilon=epsilon)
    torch.manual_seed(seed)
    build = lambda: wm.MemoryNetwork(state_dim=S, action_dim=A, num_hiddens=hidden,  # noqa: E731
                                     num_hidden_layers=layers, num_gaussians=G)
    build()  # CrossEntropyMethod.build_trainer's discarded WorldModel build
    nets = [build() for _ in range(K)]
    trainers = [trainer_mod.MDNRNNTrainer(memory_network=n, params=mdn) for n in nets]
    cfg = dict(discrete=discrete, K=K, P=P, H=H, A=A, S=S, L=layers, G=G, iters=iters,
               num_elites=E, gamma=gamma, alpha=alpha, epsilon=epsilon,
               terminal_effective=nt_weight > 0, lower=lower, upper=upper)
    planner = cp.CEMPlannerNetwork(
        mem_net_list=nets, cem_num_iterations=iters, cem_population_size=P,
        ensemble_population_size=1, num_elites=E, plan_horizon_length=H, state_dim=S,
        action_dim=A, discrete_action=discrete, terminal_effective=nt_weight > 0, gamma=gamma,
        alpha=alpha, epsilon=epsilon,
        action_upper_bounds=None if discrete else np.array(upper, dtype=np.float64),
        action_lower_bounds=None if discrete else np.array(lower, dtype=np.float64))
    arrays = {}
    p0 = cem_oracle.initial_params(seed, K, S, A, hidden, layers, G)
    for m, net in enumerate(nets):
        for i, p in enumerate(net.mdnrnn.parameters()):
            assert torch.equal(p.detach(), p0[m][i]), (name, m, i)
            arrays[f"p0.{m}.{i}.sha256"] = digest(p)
    rng = np.random.RandomState(seed + 100)
    state = rng.standard_normal(S).astype(np.float32)
    P64 = [[p.double() for p in ps] for ps in p0]
    noise, orc = cem_oracle.guard_noise(P64, cfg, state.astype(np.float64),
                                        cem_oracle.make_noise(rng, cfg), rng)
    with torch.no_grad():
        res = _run_reference_planner(planner, cp, noise, state, cfg)
    _check_against_oracle(res, orc, cfg)
    arrays["state"] = state
    for k, v in noise.items():
        arrays[f"noise.{k}"] = v
    for k, v in res.items():
        arrays[k] = v
    meta = dict(kind="cem", discrete=discrete, K=K, S=S, A=A, H=H, P=P, iters=iters,
                num_elites=E, gamma=gamma, alpha=alpha, epsilon=epsilon, hidden=hidden,
                layers=layers, G=G, not_terminal_weight=nt_weight, seed=seed,
                n_iters=int(len(res["values"])), lower=lower, upper=upper, trainer=trainer,
                lr=mdn.learning_rate)
    if trainer:
        for t in trainers:
            t.trainer = None
        tr = cem_trainer_mod.CEMTrainer(cem_planner_network=planner, world_model_trainers=trainers,
                                        parameters=cem)
        opts = tr.configure_optimizers()
        assert len(opts) == K
        gen = torch.Generator().manual_seed(seed + 1000)
        losses = []
        for it in range(N_UPDATES):
            if discrete:
                act = torch.nn.functional.one_hot(torch.randint(A, (TRAIN_T, TRAIN_B), generator=gen), A).float()
            else:
                act = torch.rand(TRAIN_T, TRAIN_B, A, generator=gen) * 2 - 1
            b = dict(state=torch.randn(TRAIN_T, TRAIN_B, S, generator=gen), action=act,
                     next_state=torch.randn(TRAIN_T, TRAIN_B, S, generator=gen),
                     reward=torch.randn(TRAIN_T, TRAIN_B, generator=gen),
                     not_terminal=(torch.rand(TRAIN_T, TRAIN_B, generator=gen) >= 0.1).float())
            for k, v in b.items():
                arrays[f"batch{it}.{k}"] = _np(v).copy()
            batch = rlt.MemoryNetworkInput(
                state=rlt.FeatureData(float_features=b["state"]),
                next_state=rlt.FeatureData(float_features=b["next_state"]),
                action=rlt.FeatureData(float_features=b["action"]), reward=b["reward"],
                not_terminal=b["not_terminal"], time_diff=None, step=None)
            losses.append(run_update(tr, batch, it, opts))
            for m, net in enumerate(nets):
                for i, p in enumerate(net.mdnrnn.parameters()):
                    arrays[f"p{it + 1}.{m}.{i}"] = _np(sample(p)).copy()
        arrays["losses"] = np.array(losses, dtype=np.float64)
        meta.update(n_updates=N_UPDATES, train_T=TRAIN_T, train_B=TRAIN_B)
    _save(name, arrays, meta)


CASES = [
    # configs/world_model/cem_cartpole_offline.yaml
    ("cem_cartpole_offline", dict(discrete=True, K=1, S=4, A=2, H=10, P=100, iters=10, E=15,
                                  gamma=1.0, hidden=100, layers=2, G=1, nt_weight=200.0, seed=0,
                                  trainer=True)),
    # cem_single_world_model_linear_dynamics_offline.yaml
    ("cem_linear_dynamics_single", dict(discrete=False, K=1, S=3, A=2, H=4, P=100, iters=10,
                                        E=15, gamma=1.0, hidden=100, layers=2, G=1,
                                        nt_weight=0.0, seed=1, lower=[-3.0, -3.0],
                                        upper=[3.0, 3.0])),
    # cem_many_world_models_linear_dynamics_offline.yaml
    ("cem_linear_dynamics_many", dict(discrete=False, K=2, S=3, A=2, H=4, P=100, iters=10,
                                      E=15, gamma=1.0, hidden=100, layers=2, G=1, nt_weight=0.0,
                                      seed=2, lower=[-3.0, -3.0], upper=[3.0, 3.0],
                                      trainer=True)),
    # odd sizes: three models, mixtures, terminals, one elite, an early stop
    ("cem_odd", dict(discrete=False, K=3, S=5, A=3, H=3, P=37, iters=10, E=1, gamma=0.9,
                     hidden=24, layers=3, G=3, nt_weight=1.0, seed=3, lower=[-1.0, 0.0, -2.0],
                     upper=[1.0, 2.0, 0.5], epsilon=0.01)),
]


def main(only=None):
    for name, kw in CASES:
        if only and name not in only:
            continue
        case(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
