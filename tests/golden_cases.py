"""The golden cases the test modules share: the names of the committed goldens of each trainer,
the oracle keyword arguments and batches they are read with, and the CRR goldens' comparisons."""
import numpy as np
import torch

from oracle import crr_oracle as CO
from tests import golden_util as G
from tests.golden_util import TOL

DQN_CASES = ["dqn_huber_double", "dqn_mse_single_masked", "dqn_sarsa", "dqn_multistep_boost",
             "dqn_timediff_odd_dims", "dqn_dueling_double", "dqn_dueling_mse_masked",
             "dqn_cartpole_config0"]


def _dqn_kwargs(meta, batch):
    kw = dict(double_q=meta["double_q"], maxq=meta["maxq"], loss=meta["loss"])
    if meta["multi_steps"] is not None:
        kw["discount_src"] = batch["step"]
    elif meta["time_diff"]:
        kw["discount_src"] = batch["time_diff"]
    if meta["boost"]:
        rb = torch.zeros(1, meta["A"])
        for k, v in meta["boost"].items():
            rb[0, int(k)] = v
        kw["reward_boost"] = rb
    return kw


SAC_CASES = ["sac_twin_alpha", "sac_single_fixed_alpha", "sac_twin_odd_dims"]


TD3_CASES = ["td3_twin", "td3_single"]


QRDQN_CASES = ["qrdqn_double", "qrdqn_single_masked", "qrdqn_sarsa_multistep", "qrdqn_dueling"]


PDQN_CASES = ["pdqn_double_mse", "pdqn_sarsa_huber_reward", "pdqn_single_multistep"]


C51_CASES = ["c51_double", "c51_single_masked_boost", "c51_sarsa_multistep"]


def _c51_kwargs(meta, batch):
    kw = dict(num_atoms=meta["N"], qmin=meta["qmin"], qmax=meta["qmax"], double_q=meta["double_q"],
              maxq=meta["maxq"])
    if meta["multi_steps"] is not None:
        kw["discount_src"] = batch["step"]
    if meta["boost"]:
        rb = torch.zeros(1, meta["A"])
        for k, v in meta["boost"].items():
            rb[0, int(k)] = v
        kw["reward_boost"] = rb
    return kw


DQN_CPE_CASES = ["dqn_cpe_huber", "dqn_cpe_mse_sarsa_multistep"]


BCQ_DQN_CASES = ["dqn_bcq_huber_double", "dqn_bcq_cpe_mse_single",
                 "dqn_bcq_dueling_multistep_boost"]


CRR_CASES = ["crr_twin_default", "crr_single_target_actor", "crr_dueling_delayed",
             "crr_entropy_clip", "crr_noise_saturated", "crr_cpe_boost", "crr_adamw_amsgrad",
             "crr_odd_dims", "crr_cartpole_manager"]


SOURCES = ("actor", "q1", "q2", "r", "c")  # the order the compact case seeds its networks in


def net_names(meta):
    """Golden prefixes of the trained networks and of their targets."""
    src = ["actor", "q1"] + (["q2"] if meta["twin"] else [])
    tgt = ["actor_t", "q1_t"] + (["q2_t"] if meta["twin"] else [])
    if meta["cpe_metrics"] is not None:
        src += ["r", "c"]
        tgt += ["ct"]
    return src, tgt


def net_dims(meta, name):
    A = meta["A"]
    out = A if name in ("actor", "q1", "q2") else (len(meta["cpe_metrics"]) + 1) * A
    return [meta["S"]] + meta["sizes"] + [out]


def initial_tensors(arrays, meta, name):
    """[W0, b0, W1, b1, ...] of network `name` before the first update (a target starts as a copy
    of its network in the compact case, whose parameters are seeded rather than stored)."""
    if not meta["compact"]:
        return [torch.from_numpy(x.copy()) for pair in G.net_pairs(arrays, name + "0") for x in pair]
    src = {"actor_t": "actor", "q1_t": "q1", "q2_t": "q2", "ct": "c"}.get(name, name)
    dims = net_dims(meta, src)
    shapes = []
    for i in range(len(dims) - 1):
        shapes += [torch.empty(dims[i + 1], dims[i]), torch.empty(dims[i + 1])]
    present = [n for n in SOURCES if n in net_names(meta)[0]]
    return CO.seeded_like(shapes, meta["seed"] + 100 + present.index(src))


def noise_of(arrays, it, which, device="cpu"):
    k = f"noise{it}.{which}"
    return torch.from_numpy(arrays[k].copy()).to(device) if k in arrays else None


def check_params(arrays, meta, name, params, tol=TOL):
    """`params` ([W0, b0, ...] tensors) against the golden's final values of network `name`."""
    if meta["compact"]:
        for i, p in enumerate(params):
            assert G.rel_err(CO.digest(p), arrays[f"{name}N.digest{i}"]) < tol, (name, i)
        return
    ref = [x for pair in G.net_pairs(arrays, name + "N") for x in pair]
    assert len(ref) == len(params)
    for i, (p, r) in enumerate(zip(params, ref)):
        assert G.rel_err(p, r) < tol, (name, i)


def check_grads(arrays, meta, opt_idx, grads, tol=TOL):
    for i, g in enumerate(grads):
        ref = arrays[f"grad0.opt{opt_idx}.{i}"]
        assert G.rel_err(CO.digest(g) if meta["compact"] else g, ref) < tol, (opt_idx, i)


def check_losses(arrays, it, losses, tol=TOL):
    ref = arrays["losses"][it]
    assert len(losses) == len(ref)
    for l, r in zip(losses, ref):
        if np.isnan(r):
            assert l is None
        else:
            assert abs(float(l) - r) <= tol * max(1.0, abs(r)), (it, float(l), r)


BC_CASES = ["bc_reference_4x4", "bc_a16_random_masks", "bc_a40_tanh_leaky"]


def golden_batch(arrays, prefix, device="cpu"):
    return {k: torch.from_numpy(arrays[f"{prefix}.{k}"].copy()).to(device)
            for k in ("state", "action", "possible_actions_mask")}


E2E = dict(S=16, A=6, B=512, sizes=[64, 64], lr=1e-2, steps=300, thr=0.3)


# share of held-out rows on which the BCQ filter keeps the behaviour action: the CPU oracle
# reaches 0.982 on these data (the misses are states next to a decision boundary of the rule);
# the bound leaves room for another arithmetic's rounding to compound over 300 Adam steps
E2E_MIN_BEHAVIOUR_KEPT = 0.95


# and the filter does narrow the mask (the oracle keeps 0.17 of all (row, action) pairs)
E2E_MAX_KEPT = 0.3


def e2e_data(seed=0):
    """(behaviour map, train batches, held-out states): the logged action of a state is
    argmax(state @ Wb), every action is possible."""
    g = torch.Generator().manual_seed(seed)
    S, A, B = E2E["S"], E2E["A"], E2E["B"]
    Wb = torch.randn(S, A, generator=g)
    batches = []
    for _ in range(E2E["steps"]):
        x = torch.randn(B, S, generator=g)
        batches.append(dict(state=x, action=torch.nn.functional.one_hot((x @ Wb).argmax(1), A).float(),
                            possible_actions_mask=torch.ones(B, A)))
    held_out = torch.randn(B, S, generator=g)
    return Wb, batches, held_out


def e2e_metrics(keep, Wb, states):
    """(share of rows whose behaviour action the BCQ keep-mask holds, share of all pairs kept)."""
    beh = (states @ Wb).argmax(1)
    return float(keep[torch.arange(len(beh)), beh].mean()), float(keep.mean())


SAC_VALUE_CASES = ["sac_value_twin_alpha", "sac_value_single_prior", "sac_value_fixed_alpha_odd",
                   "sac_crr_exponent", "sac_crr_indicator", "sac_pendulum_manager",
                   "sac_crr_pendulum_manager"]


def opt_names(meta):
    """Optimizer order of the reference (sac_trainer.py:148-193)."""
    return (["q1"] + (["q2"] if meta["twin"] else []) + ["actor"]
            + (["alpha"] if meta["learn_alpha"] else []) + ["value"])


INPUTMAKER_CASES = ["inputmaker_parametric_uniform_terminal", "inputmaker_parametric_h3_wrap",
                    "inputmaker_parametric_masks_logprob", "inputmaker_parametric_per"]


CARTPOLE_CASES = ["pdqn_adamw_amsgrad_cartpole", "pdqn_sarsa_adam_cartpole"]


def cartpole_batch(arrays, it, device="cpu"):
    """The batch of update `it` of a make_parametric_golden.py CartPole case."""
    pre = f"batch{it}."
    return {k[len(pre):]: torch.from_numpy(v.copy()).to(device)
            for k, v in arrays.items() if k.startswith(pre)}


def batch_at(arrays, it, device="cpu"):
    """The batch of update `it` of a make_adamw_golden.py case."""
    pre = f"batch{it}."
    return {k[len(pre):]: torch.from_numpy(v.copy()).to(device)
            for k, v in arrays.items() if k.startswith(pre)}
