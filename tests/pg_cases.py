"""Shared helpers of the policy-gradient tests: the goldens of oracle/make_pg_golden.py as
trajectories, oracle networks and replays of the reference's updates."""
import numpy as np
import torch

from oracle import pg_oracle as PO
from oracle import td_oracle as O
from tests import golden_util as G

REINFORCE_CASES = ["pg_reinforce_cartpole", "pg_reinforce_whiten_offpolicy",
                   "pg_reinforce_baseline", "pg_reinforce_gamma0_constant"]
PPO_CASES = ["pg_ppo_cartpole", "pg_ppo_baseline_entropy_dueling", "pg_ppo_td_next_state",
             "pg_ppo_td_no_next_state", "pg_ppo_whiten_constant"]
PG_CASES = REINFORCE_CASES + PPO_CASES
FIELDS = ("state", "action", "reward", "log_prob", "possible_actions_mask", "next_state",
          "not_terminal")


def trajectories(arrays, device="cpu"):
    out, k = [], 0
    while f"traj{k}.state" in arrays:
        out.append({f: torch.from_numpy(arrays[f"traj{k}.{f}"].copy()).to(device)
                    for f in FIELDS if f"traj{k}.{f}" in arrays})
        k += 1
    return out


def as_input(d):
    from reagent_b200.core import types as rlt

    return rlt.PolicyGradientInput(
        state=rlt.FeatureData(d["state"]), action=d["action"], reward=d["reward"],
        log_prob=d["log_prob"], possible_actions_mask=d.get("possible_actions_mask"),
        next_state=rlt.FeatureData(d["next_state"]) if "next_state" in d else None,
        not_terminal=d.get("not_terminal"))


def policy_acts(meta):
    return list(meta["acts"]) + ["linear"]


def value_acts(meta):
    return ["relu"] * len(meta["value_sizes"]) + ["linear"]


def oracle_nets(arrays, meta, u=0):
    pol = G.oracle_net(arrays, f"policy{u}", policy_acts(meta), requires_grad=True)
    val = None
    if meta["value_sizes"] is not None:
        val = G.oracle_net(arrays, f"value{u}", value_acts(meta), requires_grad=True)
    return pol, val


def adam(meta, net):
    return None if net is None else O.AdamState(O.net_params(net), lr=meta["lr"],
                                                weight_decay=meta["wd"])


def minibatches(arrays, meta):
    """[(update u, [trajectory indices])] in the order the reference ran them."""
    out = []
    for u in range(meta["n_updates"]):
        base = u * meta["update_freq"]
        for e in range(meta["update_epochs"]):
            perm = arrays[f"perm{u}.{e}"]
            for i in range(0, len(perm), meta["ppo_batch_size"]):
                out.append((u, [base + int(j) for j in perm[i: i + meta["ppo_batch_size"]]]))
    return out


def reinforce_kwargs(meta):
    return {k: meta[k] for k in ("gamma", "off_policy", "reward_clip", "clip_param", "normalize",
                                 "subtract_mean", "offset_clamp_min", "temperature")}


def ppo_kwargs(meta):
    return {k: meta[k] for k in ("gamma", "reward_clip", "normalize", "subtract_mean",
                                 "offset_clamp_min", "td_error_advantage", "ppo_epsilon",
                                 "entropy_weight", "temperature")}


def value_head_free(meta, n_params):
    """Indices of the parameters whose update is rounding residue: the value head of a dueling
    policy.  The softmax does not change when V shifts every score, so the true gradient of that
    head is 0; Adam normalises whatever residue each side computes into steps of up to lr, so
    those parameters are not compared.  Empty for a plain policy."""
    return set(range(n_params - 4, n_params)) if meta["dueling"] else set()


def check_net(arrays, prefix, params, tol=G.TOL, skip=()):
    """params in parameter order against the dumped network `prefix`."""
    pairs = G.net_pairs(arrays, prefix)
    flat = [x for w, b in pairs for x in (w, b)]
    assert len(flat) == len(params), (prefix, len(flat), len(params))
    for i, (p, want) in enumerate(zip(params, flat)):
        if i in skip:
            continue
        err = G.rel_err(p, want)
        assert err < tol, (prefix, i, err)


def check_grads(arrays, opt_idx, grads, tol=G.TOL):
    """Each gradient within `tol` of the reference's, relative to its own largest entry.  A
    tensor whose reference is below 1e-6 of the network's largest entry is a true 0 (the value
    head of a dueling policy, see value_head_free): it must stay below tol of that entry."""
    refs = [arrays[f"grad0.opt{opt_idx}.{i}"] for i in range(len(grads))]
    scale = max(float(np.abs(r).max()) for r in refs)
    for i, (g, r) in enumerate(zip(grads, refs)):
        g = torch.as_tensor(g, dtype=torch.float64).cpu()
        if float(np.abs(r).max()) < 1e-6 * scale:
            assert float(g.abs().max()) < tol * scale, (f"grad0.opt{opt_idx}.{i}", "not 0")
            continue
        err = G.rel_err(g, r)
        assert err < tol, (f"grad0.opt{opt_idx}.{i}", err)


def check_losses(got, want, tol=G.TOL):
    for g, w in zip(got, want):
        assert abs(g - w) <= tol * max(1.0, abs(w)), (got, list(want))
