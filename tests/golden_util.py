"""Helpers to read tests/golden/*.npz (produced by oracle/make_golden.py from the reference)."""
import json
import os

import numpy as np
import torch

TOL = 1e-5  # the project's parity bar
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(bytes(z["__meta__"]).decode())
    arrays = {k: z[k] for k in z.files if k != "__meta__"}
    return arrays, meta


def oracle_net(arrays, prefix, acts, requires_grad=False):
    if f"{prefix}.shared.W0" in arrays:
        # DuelingQNetwork.make_fully_connected (dueling_q_network.py:48-90): the shared trunk ends
        # in a linear layer; both heads are [E -> E/2 (last activation) -> out (linear)]
        head = [acts[-2], "linear"]
        return {"kind": "dueling",
                "shared": oracle_net(arrays, prefix + ".shared", list(acts[:-2]) + ["linear"], requires_grad),
                "adv": oracle_net(arrays, prefix + ".advantage", head, requires_grad),
                "val": oracle_net(arrays, prefix + ".value", head, requires_grad)}
    W, b = [], []
    i = 0
    while f"{prefix}.W{i}" in arrays:
        W.append(torch.from_numpy(arrays[f"{prefix}.W{i}"].copy()).requires_grad_(requires_grad))
        b.append(torch.from_numpy(arrays[f"{prefix}.b{i}"].copy()).requires_grad_(requires_grad))
        i += 1
    return {"W": W, "b": b, "act": list(acts)}


def net_pairs(arrays, prefix):
    """[(W, b)] arrays of a dumped network in parameter order (dueling: shared, advantage, value)."""
    if f"{prefix}.shared.W0" in arrays:
        return sum((net_pairs(arrays, f"{prefix}.{part}") for part in ("shared", "advantage", "value")), [])
    out, i = [], 0
    while f"{prefix}.W{i}" in arrays:
        out.append((arrays[f"{prefix}.W{i}"], arrays[f"{prefix}.b{i}"]))
        i += 1
    return out


def load_into_module(arrays, prefix, module):
    """Copy golden weights into a reagent_b200 model (module.fc.dnn[i][0] Linear views)."""
    if hasattr(module, "shared_network"):
        for part in ("shared", "advantage", "value"):
            load_into_module(arrays, f"{prefix}.{part}", getattr(module, part + "_network"))
        return
    fc = module.fc if hasattr(module, "fc") else module
    with torch.no_grad():
        for i, seq in enumerate(fc.dnn):
            seq[0].weight.copy_(torch.from_numpy(arrays[f"{prefix}.W{i}"]))
            seq[0].bias.copy_(torch.from_numpy(arrays[f"{prefix}.b{i}"]))


def batch_tensors(arrays, device="cpu"):
    return {k[len("batch."):]: torch.from_numpy(v.copy()).to(device)
            for k, v in arrays.items() if k.startswith("batch.")}


def rel_err(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def grad_close(g_gpu, g_ref, what="grad", l2_tol=1e-3, max_tol=1e-2):
    """Gradient agreement at BASELINE config sizes.  The forward activations agree to ~5e-6
    (3xTF32 tensor-core products carry ~22 mantissa bits); a hidden unit whose pre-activation
    is within that distance of 0 gets the other ReLU mask, which changes one row of that
    layer's weight gradient by O(|x|/B) while everything else agrees to ~1e-5 (the golden-size
    cases, where no unit sits that close to 0, hold 1e-5 on every element).  Hence a relative
    L2 bound (measured <= 5e-4) plus a max-norm bound."""
    a = torch.as_tensor(g_gpu, dtype=torch.float64).cpu().reshape(-1)
    b = torch.as_tensor(g_ref, dtype=torch.float64).cpu().reshape(-1)
    l2 = float((a - b).norm() / (b.norm() + 1e-30))
    mx = float((a - b).abs().max() / (b.abs().max() + 1e-30))
    assert l2 < l2_tol, (what, "rel L2", l2)
    assert mx < max_tol, (what, "rel max", mx)
    return l2, mx


def _cmp_net(net, arrays, prefix, tol):
    for i in range(len(net["W"])):
        assert rel_err(net["W"][i], arrays[f"{prefix}.W{i}"]) < tol, f"{prefix}.W{i}"
        assert rel_err(net["b"][i], arrays[f"{prefix}.b{i}"]) < tol, f"{prefix}.b{i}"


def _cmp_losses(got, want, tol):
    for g, w in zip(got, want):
        if g is None:
            assert np.isnan(w)
        else:
            assert abs(g - w) <= tol * max(1.0, abs(w)), (got, want)


def _cmp_module(mod, arrays, prefix, tol=TOL):
    for i, seq in enumerate(mod.fc.dnn):
        assert rel_err(seq[0].weight, arrays[f"{prefix}.W{i}"]) < tol, f"{prefix}.W{i}"
        assert rel_err(seq[0].bias, arrays[f"{prefix}.b{i}"]) < tol, f"{prefix}.b{i}"


def _adam_close(w_gpu, w_ref, meta):
    """Post-Adam parameters at config sizes: every element within the total step budget
    (n_updates * 2 * lr) and the typical element within 2 % of one step."""
    d = (w_gpu.detach().cpu().double() - w_ref.detach().double()).abs()
    assert float(d.max()) <= 2.0 * meta["n_updates"] * meta["lr"] * 1.01
    assert float(d.median()) < 0.02 * meta["lr"], float(d.median())
