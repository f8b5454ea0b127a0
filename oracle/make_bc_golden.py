"""Generate the behavioral-cloning golden vectors in tests/golden/ by running the UNMODIFIED
reference BehavioralCloningTrainer through oracle/ref_harness.py.  Needs the reference checkout
(build container only); the files are committed.

    python oracle/make_bc_golden.py            # regenerate every BC case
    python oracle/make_bc_golden.py NAME ...   # only the named ones

The reference labels row i with `labels.max(dim=0)[1][i]`, the row whose one-hot sits in column
i.  That is row i's own action only when B == A and the label matrix is an involutive
permutation, so every case here is of that kind and the script asserts it.  Each file holds
  q0.W*/b*                    initial bc_net weights
  batch{t}.state/action/possible_actions_mask   the batch of update t (and `val.*`)
  logits{t}                   bc_net(state, possible_actions_mask) before update t
  grad{t}.*                   parameter gradients of update t (parameters() order)
  q{t}.W*/b*                  parameters after the Adam step of update t
  losses                      the yielded loss of each update
  val_loss                    validation_step on `val.*` after the last update
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import N_UPDATES, _dump_net, _np, _perturb, _save  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402


def _involution(n, n_fixed, gen):
    """A random permutation p with p[p[i]] == i and `n_fixed` fixed points."""
    order = torch.randperm(n, generator=gen).tolist()
    p = list(range(n))
    rest = order[n_fixed:]
    assert len(rest) % 2 == 0
    for i in range(0, len(rest), 2):
        a, b = rest[i], rest[i + 1]
        p[a], p[b] = b, a
    return torch.tensor(p)


def _reference_test_batch(gen):
    """get_dummy_batch of reagent/test/training/test_behavioral_cloning.py (one-hot identity
    labels as int64, the mask keeping each label and one neighbour, noisy states)."""
    action = torch.tensor([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    mask = torch.tensor([[1, 1, 0, 0], [0, 1, 1, 0], [0, 0, 1, 1], [1, 0, 0, 1]])
    state = torch.tensor([
        [+0.1, +0.2, +0.3, +0.4, +0.5, +0.6, +0.7, +0.8],
        [+0.1, +0.2, +0.3, +0.4, -0.5, -0.6, -0.7, -0.8],
        [-0.1, -0.2, -0.3, -0.4, +0.5, +0.6, +0.7, +0.8],
        [-0.1, -0.2, -0.3, -0.4, -0.5, -0.6, -0.7, -0.8]])
    state = state + (1e-8 ** 0.5) * torch.rand(state.shape, generator=gen)
    return dict(state=state, action=action, possible_actions_mask=mask)


def _random_batch(gen, A, S, n_fixed, p_masked):
    labels = _involution(A, n_fixed, gen)
    action = torch.nn.functional.one_hot(labels, A).float()
    mask = (torch.rand(A, A, generator=gen) > p_masked).float()
    mask[torch.arange(A), labels] = 1.0
    return dict(state=torch.randn(A, S, generator=gen), action=action, possible_actions_mask=mask)


def bc_case(name, *, S, A, sizes, acts, lr, seed, make_batch):
    rlt = ref("reagent.core.types")
    dqn_mod = ref("reagent.models.dqn")
    bct = ref("reagent.training.behavioral_cloning_trainer")
    union = ref("reagent.optimizer.union")
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed)
    net = dqn_mod.FullyConnectedDQN(S, A, list(sizes), list(acts))
    _perturb(net)
    trainer = bct.BehavioralCloningTrainer(
        bc_net=net, optimizer=union.Optimizer__Union(Adam=union.classes["Adam"](lr=lr)))
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    assert len(opts) == 1
    arrays = {}
    _dump_net(arrays, "q0", net)
    losses = []
    for it in range(N_UPDATES):
        b = make_batch(gen)
        B = b["state"].shape[0]
        # the reference's dim-0 labels equal every row's own action on this batch
        assert B == A and torch.equal(b["action"].max(dim=0)[1], b["action"].argmax(dim=1)), name
        for k, v in b.items():
            arrays[f"batch{it}.{k}"] = _np(v).copy()
        batch = rlt.BehavioralCloningModelInput(
            state=rlt.FeatureData(float_features=b["state"]), action=b["action"],
            possible_actions_mask=b["possible_actions_mask"])
        with torch.no_grad():
            arrays[f"logits{it}"] = _np(net(batch.state, possible_actions_mask=b["possible_actions_mask"]))
        cap = {}
        out = run_update(trainer, batch, it, opts, capture=cap)
        losses.append(out[0])
        for i, g in enumerate(cap[0]):
            arrays[f"grad{it}.{i}"] = _np(g)
        _dump_net(arrays, f"q{it + 1}", net)
    vb = make_batch(gen)
    assert torch.equal(vb["action"].max(dim=0)[1], vb["action"].argmax(dim=1)), name
    for k, v in vb.items():
        arrays[f"val.{k}"] = _np(v).copy()
    val = trainer.validation_step(rlt.BehavioralCloningModelInput(
        state=rlt.FeatureData(float_features=vb["state"]), action=vb["action"],
        possible_actions_mask=vb["possible_actions_mask"]), 0)
    arrays["losses"] = np.array(losses, dtype=np.float64)
    arrays["val_loss"] = np.array(float(val), dtype=np.float64)
    _save(name, arrays, dict(kind="bc", S=S, A=A, sizes=list(sizes), acts=list(acts), lr=lr,
                             n_updates=N_UPDATES))


CASES = [
    # the reference test's own data and network
    ("bc_reference_4x4", dict(S=8, A=4, sizes=(7, 6, 5), acts=("relu",) * 3, lr=1e-2, seed=0,
                              make_batch=_reference_test_batch)),
    # 16 actions, pairs swapped plus fixed points, random masks that keep the labels
    ("bc_a16_random_masks", dict(S=12, A=16, sizes=(32, 24), acts=("relu", "relu"), lr=1e-2,
                                 seed=1, make_batch=lambda g: _random_batch(g, 16, 12, 4, 0.4))),
    # 40 actions: rows wider than a warp
    ("bc_a40_tanh_leaky", dict(S=10, A=40, sizes=(48, 32), acts=("tanh", "leaky_relu"), lr=5e-3,
                               seed=2, make_batch=lambda g: _random_batch(g, 40, 10, 6, 0.3))),
]


def main(only=None):
    for name, kw in CASES:
        if only and name not in only:
            continue
        bc_case(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
