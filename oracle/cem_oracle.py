"""Plain-numpy/torch restatement of the cross-entropy-method planner (reagent/models/
cem_planner.py CEMPlannerNetwork) in fp64, given the planner's noise.  Each planned step is the
fp64 T = 1 forward of oracle.mdnrnn_oracle from a zero state, as the reference calls the world
model with a [1, 1, .] input and no hidden state.

Noise (numpy arrays, the layout of reagent_b200.models.CEMNoise):
  model_idx  int   [iters, P]           world model of each trajectory
  action_idx int   [P, H]               discrete: the action of each step
  truncnorm  fp64  [iters, P, H * A]    continuous: truncnorm(-2, 2) draws
  step       fp32  [iters, P, H, S + 2] mixture uniform | S standard normals | Bernoulli uniform
The draws are the reference's, written as formulas of the noise:
  mixture    k = the first k with u * sum(p) < cumsum(p)_k, p = exp(logpi)
  next state mus[k] + sigmas[k] * z
  terminal   not_terminal = u < sigmoid(not_terminal logit)  (only with terminal_effective)
  truncnorm  ndtri(Phi(-2) + u * (Phi(2) - Phi(-2)))

`plan` also reports every decision that lies near a boundary, where an fp32 planner could
decide otherwise: a mixture or Bernoulli uniform within 1e-4 of its threshold, a gap between
the num_elites-th and the next value below 1e-3 relative, or a best first-action ratio within
1e-6 of the runner-up.  `guard_noise` redraws the numbers behind such decisions until there is
none, so comparisons of a float32 planner with this oracle at 1e-5 are well-posed.
"""
import math

import numpy as np
import torch
from scipy.special import ndtri

from oracle import mdnrnn_oracle as mo

PHI_LO = 0.5 * math.erfc(math.sqrt(2.0))
PHI_WIDTH = math.erf(math.sqrt(2.0))
U_MARGIN, GAP_REL, RATIO_MARGIN = 1e-4, 1e-3, 1e-6
CONTINUOUS_TRAINING_ACTION_RANGE = (-1.0, 1.0)


def initial_params(seed, num_models, state_dim, action_dim, hidden, layers, gaussians):
    """The seeded initial parameters of the num_models world models that
    CrossEntropyMethod.build_trainer makes under torch.manual_seed(seed): one MemoryNetwork
    built and discarded, then num_models more, each as mdnrnn_oracle.initial_params builds it."""
    torch.manual_seed(seed)
    out = []
    for m in range(num_models + 1):
        rnn = torch.nn.LSTM(state_dim + action_dim, hidden, layers)
        head = torch.nn.Linear(hidden, (2 * state_dim + 1) * gaussians + 2)
        if m > 0:
            out.append([p.detach().clone() for p in list(rnn.parameters()) + list(head.parameters())])
    return out


def make_noise(rng: np.random.RandomState, cfg):
    """Fresh noise of the planner shape `cfg` from a numpy generator."""
    iters = 1 if cfg["discrete"] else cfg["iters"]
    P, H, A, S = cfg["P"], cfg["H"], cfg["A"], cfg["S"]
    step = np.empty((iters, P, H, S + 2), dtype=np.float32)
    step[..., 0] = rng.uniform(size=(iters, P, H))
    step[..., 1:S + 1] = rng.standard_normal((iters, P, H, S))
    step[..., S + 1] = rng.uniform(size=(iters, P, H))
    noise = dict(model_idx=rng.randint(0, cfg["K"], size=(iters, P)).astype(np.int32), step=step)
    if cfg["discrete"]:
        noise["action_idx"] = rng.randint(0, A, size=(P, H)).astype(np.int32)
    else:
        noise["truncnorm"] = ndtri(PHI_LO + rng.uniform(size=(iters, P, H * A)) * PHI_WIDTH)
    return noise


def _rollout(params, cfg, state, actions, model_idx, step_noise, it, violations):
    """Values [P] (fp64) of one iteration's trajectories; actions fp64 [P, H, A]."""
    P, H, S, G = cfg["P"], cfg["H"], cfg["S"], cfg["G"]
    values = np.zeros(P)
    for m, P_m in enumerate(params):
        rows = np.nonzero(model_idx == m)[0]
        if len(rows) == 0:
            continue
        x = np.tile(np.asarray(state, dtype=np.float64), (len(rows), 1))
        alive = np.ones(len(rows), dtype=bool)
        for j in range(H):
            out = mo.forward(P_m, torch.from_numpy(x)[None], torch.from_numpy(actions[rows, j])[None],
                             cfg["L"], G)
            mus, sig = out["mus"][0].numpy(), out["sigmas"][0].numpy()
            logpi, rw, nt = out["logpi"][0].numpy(), out["reward"][0].numpy(), out["not_terminal"][0].numpy()
            nz = step_noise[it, rows, j].astype(np.float64)
            p = np.exp(logpi)
            tot = p.sum(axis=1)
            cum = np.cumsum(p, axis=1)
            thr = nz[:, 0] * tot
            k = np.argmax(thr[:, None] < cum, axis=1)
            k[~(thr[:, None] < cum).any(axis=1)] = G - 1
            if G > 1:
                near = np.abs(cum[:, :-1] / tot[:, None] - nz[:, :1]).min(axis=1) < U_MARGIN
                for i in np.nonzero(near & alive)[0]:
                    violations.append(("mixture", it, int(rows[i]), j))
            ns = mus[np.arange(len(rows)), k] + sig[np.arange(len(rows)), k] * nz[:, 1:S + 1]
            values[rows] += np.where(alive, rw * cfg["gamma"] ** j, 0.0)
            if cfg["terminal_effective"]:
                pt = 1.0 / (1.0 + np.exp(-nt))
                u = nz[:, S + 1]
                for i in np.nonzero((np.abs(u - pt) < U_MARGIN) & alive)[0]:
                    violations.append(("terminal", it, int(rows[i]), j))
                alive = alive & (u < pt)
            x = np.where(alive[:, None], ns, x)
            if not alive.any():
                break
    return values


def _tiled_bounds(cfg):
    return (np.tile(np.asarray(cfg["lower"], dtype=np.float64), cfg["H"]),
            np.tile(np.asarray(cfg["upper"], dtype=np.float64), cfg["H"]))


def plan(params, cfg, state, noise):
    """The planner on `params` (a list of fp64 parameter lists, one per world model) from
    `state` [S].  cfg: discrete, K, P, H, A, S, L, G, iters, num_elites, gamma, alpha, epsilon,
    terminal_effective, lower / upper [A] (continuous).  Returns values [n, P], elites [n, E]
    (ascending value), mean / var [n, H*A] after each update, n_iters, action (discrete: the
    index; continuous: fp64 [A] in CONTINUOUS_TRAINING_ACTION_RANGE) and the violations."""
    P, H, A = cfg["P"], cfg["H"], cfg["A"]
    viol = []
    if cfg["discrete"]:
        acts = np.eye(A)[noise["action_idx"]]
        values = _rollout(params, cfg, state, acts, noise["model_idx"][0], noise["step"], 0, viol)
        first = noise["action_idx"][:, 0]
        cnt, tally = np.zeros(A), np.zeros(A)
        for f, v in zip(first, values):
            cnt[f] += 1
            tally[f] += v
        with np.errstate(invalid="ignore", divide="ignore"):
            ratio = tally / cnt
        best = int(np.nanargmax(ratio))
        r = np.sort(ratio[~np.isnan(ratio)])
        if len(r) > 1 and r[-1] - r[-2] < RATIO_MARGIN * max(1.0, abs(r[-1])):
            viol.append(("ratio", 0, -1, -1))
        return dict(values=values[None], n_iters=1, action=best, violations=viol)
    lb, ub = _tiled_bounds(cfg)
    mean = (ub + lb) / 2
    var = (ub - lb) ** 2 / 16
    E, al = cfg["num_elites"], cfg["alpha"]
    out = dict(values=[], elites=[], mean=[], var=[])
    for it in range(cfg["iters"]):
        cv = np.minimum(np.minimum(((mean - lb) / 2) ** 2, ((ub - mean) / 2) ** 2), var)
        sol = noise["truncnorm"][it] * np.sqrt(cv) + mean
        acts = sol.reshape(P, H, A).astype(np.float32).astype(np.float64)
        values = _rollout(params, cfg, state, acts, noise["model_idx"][it], noise["step"], it, viol)
        order = np.lexsort((np.arange(P), values))  # ascending value, ties by index
        el = order[-E:]
        if E < P:
            a, b = values[order[-E]], values[order[-E - 1]]
            if a - b < GAP_REL * max(abs(a), abs(b)):
                viol.append(("elite", it, int(order[-E]), int(order[-E - 1])))
        elites = sol[el]
        mean = al * mean + (1 - al) * np.mean(elites, axis=0)
        var = al * var + (1 - al) * np.var(elites, axis=0)
        for k, v in (("values", values), ("elites", el), ("mean", mean), ("var", var)):
            out[k].append(v)
        if np.max(var) <= cfg["epsilon"]:
            break
    out = {k: np.array(v) for k, v in out.items()}
    lo, hi = np.asarray(cfg["lower"], np.float64), np.asarray(cfg["upper"], np.float64)
    low, high = CONTINUOUS_TRAINING_ACTION_RANGE
    out.update(n_iters=len(out["values"]), violations=viol,
               action=((mean[:A] - lo) / (hi - lo)) * (high - low) + low)
    return out


def guard_noise(params, cfg, state, noise, rng: np.random.RandomState, max_rounds=500):
    """Redraw the numbers behind every near-boundary decision of `plan` until there is none.
    Returns (noise, plan result)."""
    noise = {k: v.copy() for k, v in noise.items()}
    S = cfg["S"]
    for _ in range(max_rounds):
        res = plan(params, cfg, state, noise)
        if not res["violations"]:
            return noise, res
        for kind, it, p, j in res["violations"]:
            if kind == "mixture":
                noise["step"][it, p, j, 0] = rng.uniform()
            elif kind == "terminal":
                noise["step"][it, p, j, S + 1] = rng.uniform()
            elif kind == "elite":
                for q in (p, j):
                    noise["truncnorm"][it, q] = ndtri(
                        PHI_LO + rng.uniform(size=noise["truncnorm"].shape[2]) * PHI_WIDTH)
            else:  # ratio
                noise["action_idx"][rng.randint(cfg["P"])] = rng.randint(
                    0, cfg["A"], size=cfg["H"])
    raise RuntimeError("guard_noise: no guarded noise within the round limit")
