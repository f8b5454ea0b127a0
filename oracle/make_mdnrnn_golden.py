"""Generate the MDN-RNN golden vectors in tests/golden/ by running the UNMODIFIED reference
MDNRNNTrainer (reagent/training/world_model/mdnrnn_trainer.py) through oracle/ref_harness.py.
Needs the reference checkout (build container only); the files are committed.

    python oracle/make_mdnrnn_golden.py            # regenerate every case
    python oracle/make_mdnrnn_golden.py NAME ...   # only the named ones

The reference's model manager (model_managers/model_based/world_model.py) imports pyspark, so
MemoryNetwork is built here the way its build_trainer builds it.  Two shims on the trainer
instance: configure_optimizers() returns bare optimizers (passed to run_update as `opts`), and
train_step_gen reads `self.trainer.logger` (set `trainer.trainer = None`).

A trainer case holds
  p0.{i}.sha256           SHA-256 of the seeded initial parameters, parameters() order (they
                          are rebuilt with oracle.mdnrnn_oracle.initial_params(seed, ...))
  batch{t}.{state,action,next_state,reward,not_terminal}   the batch of update t
  out.{field}             MemoryNetworkOutput of batch 0 under p0 (all eight fields), batch
                          rows [0, OUT_ROWS) only
  loss_sd.{k} / loss.{k}  get_loss(batch0) with and without state_dim, k in gmm bce mse loss
  grad.{i}                gradients of update 0           } on oracle.mdnrnn_oracle.sample's
  p{t}.{i}                parameters after update t       } strided subsample of each tensor
                                                            (file size)
  losses                  the loss yielded by each update
The `memory_input_maker` case holds the reference maker's output on ReplayBuffer samples.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import _np, _save  # noqa: E402
from oracle.mdnrnn_oracle import digest, initial_params, sample  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402

N_UPDATES = 2
OUT_ROWS = 32  # forward outputs are kept for the first 32 rows of batch 0 (file size)
OUT_FIELDS = ("mus", "sigmas", "logpi", "reward", "not_terminal", "last_step_lstm_hidden",
              "last_step_lstm_cell", "all_steps_lstm_hidden")
LOSS_KEYS = ("gmm", "bce", "mse", "loss")


def _batch(gen, T, B, S, A, discrete, p_terminal):
    if discrete:
        action = torch.nn.functional.one_hot(torch.randint(A, (T, B), generator=gen), A).float()
    else:
        action = torch.rand(T, B, A, generator=gen) * 2 - 1
    nt = (torch.rand(T, B, generator=gen) >= p_terminal).float()
    return dict(state=torch.randn(T, B, S, generator=gen), action=action,
                next_state=torch.randn(T, B, S, generator=gen),
                reward=torch.randn(T, B, generator=gen), not_terminal=nt)


def trainer_case(name, *, S, A, T, B, discrete, p_terminal=0.05, seed=0, **param_kw):
    rlt = ref("reagent.core.types")
    params_mod = ref("reagent.core.parameters")
    wm = ref("reagent.models.world_model")
    trainer_mod = ref("reagent.training.world_model.mdnrnn_trainer")
    params = params_mod.MDNRNNTrainerParameters(action_dim=A, **param_kw)
    torch.manual_seed(seed)
    net = wm.MemoryNetwork(state_dim=S, action_dim=A, num_hiddens=params.hidden_size,
                           num_hidden_layers=params.num_hidden_layers,
                           num_gaussians=params.num_gaussians)
    trainer = trainer_mod.MDNRNNTrainer(memory_network=net, params=params)
    trainer.trainer = None
    opts = trainer.configure_optimizers()
    assert len(opts) == 1
    gen = torch.Generator().manual_seed(seed + 1000)
    arrays = {}
    p0 = initial_params(seed, S, A, params.hidden_size, params.num_hidden_layers,
                        params.num_gaussians)
    for i, p in enumerate(net.mdnrnn.parameters()):
        assert torch.equal(p.detach(), p0[i]), (name, i)
        arrays[f"p0.{i}.sha256"] = digest(p)

    def to_input(b):
        return rlt.MemoryNetworkInput(
            state=rlt.FeatureData(float_features=b["state"]),
            next_state=rlt.FeatureData(float_features=b["next_state"]),
            action=rlt.FeatureData(float_features=b["action"]), reward=b["reward"],
            not_terminal=b["not_terminal"], time_diff=None, step=None)

    losses = []
    for it in range(N_UPDATES):
        b = _batch(gen, T, B, S, A, discrete, p_terminal)
        for k, v in b.items():
            arrays[f"batch{it}.{k}"] = _np(v).copy()
        batch = to_input(b)
        if it == 0:
            with torch.no_grad():
                out = net(batch.state, batch.action)
                for f in OUT_FIELDS:
                    v = getattr(out, f)
                    rows = v[:, :OUT_ROWS]  # batch is dim 1 of every field
                    arrays[f"out.{f}"] = _np(rows).copy()
                for key, sd in (("loss_sd", S), ("loss", None)):
                    ls = trainer.get_loss(batch, sd)
                    for k in LOSS_KEYS:
                        arrays[f"{key}.{k}"] = np.array(float(ls[k]), dtype=np.float64)
        cap = {}
        out = run_update(trainer, batch, it, opts, capture=cap)
        losses.append(out[0])
        if it == 0:
            for i, g in enumerate(cap[0]):
                arrays[f"grad.{i}"] = _np(sample(g)).copy()
        for i, p in enumerate(net.mdnrnn.parameters()):
            arrays[f"p{it + 1}.{i}"] = _np(sample(p)).copy()
    arrays["losses"] = np.array(losses, dtype=np.float64)
    meta = dict(kind="mdnrnn", S=S, A=A, T=T, B=B, H=params.hidden_size,
                L=params.num_hidden_layers, G=params.num_gaussians, lr=params.learning_rate,
                next_state_weight=params.next_state_loss_weight,
                not_terminal_weight=params.not_terminal_loss_weight,
                reward_weight=params.reward_loss_weight,
                fit_only_one_next_step=params.fit_only_one_next_step, n_updates=N_UPDATES,
                seed=seed)
    _save(name, arrays, meta)


def input_maker_case(name="memory_input_maker", seed=7):
    """The reference maker on ReplayBuffer(stack_size=3, return_everything_as_stack=True)
    samples, discrete and continuous, with terminals inside the stack window."""
    crb = ref("reagent.replay_memory.circular_replay_buffer")
    tp = ref("reagent.gym.preprocessors.trainer_preprocessor")
    arrays = {}
    for kind, num_actions in (("discrete", 3), ("continuous", None)):
        np.random.seed(seed)
        S, N, B = 4, 40, 8
        rb = crb.ReplayBuffer(stack_size=3, replay_capacity=64, batch_size=B,
                              return_everything_as_stack=True)
        rng = np.random.RandomState(seed)
        adds = dict(observation=rng.randn(N, S).astype(np.float32),
                    action=(rng.randint(num_actions, size=N) if num_actions
                            else rng.uniform(-1, 1, (N, 2)).astype(np.float32)),
                    reward=rng.randn(N).astype(np.float32),
                    terminal=(rng.rand(N) < 0.2).astype(np.uint8))
        adds["terminal"][[5, 6, 13]] = 1
        for i in range(N):
            rb.add(observation=adds["observation"][i], action=adds["action"][i],
                   reward=adds["reward"][i], terminal=adds["terminal"][i])
        for k, v in adds.items():
            arrays[f"{kind}.add.{k}"] = np.asarray(v)
        idx = np.array([3, 7, 8, 14, 15, 20, 31, 36], dtype=np.int64)
        sample = rb.sample_transition_batch(batch_size=B, indices=torch.from_numpy(idx))
        for f in ("state", "action", "reward", "next_state", "terminal"):
            arrays[f"{kind}.sample.{f}"] = _np(getattr(sample, f)).copy()
        arrays[f"{kind}.indices"] = idx
        out = tp.MemoryNetworkInputMaker(num_actions)(sample)
        for f, v in (("state", out.state.float_features), ("action", out.action.float_features),
                     ("next_state", out.next_state.float_features), ("reward", out.reward),
                     ("not_terminal", out.not_terminal)):
            arrays[f"{kind}.out.{f}"] = _np(v).copy()
    _save(name, arrays, dict(kind="memory_input_maker", stack_size=3))


CASES = [
    # configs/world_model/cartpole_features.yaml
    ("mdnrnn_cartpole_features", dict(S=4, A=2, T=1, B=1024, discrete=True, hidden_size=50,
                                      num_hidden_layers=2, num_gaussians=1, seed=0)),
    # the mdnrnn block of configs/world_model/cem_cartpole_offline.yaml
    ("mdnrnn_cem_cartpole", dict(S=4, A=2, T=1, B=1024, discrete=True, hidden_size=100,
                                 num_hidden_layers=2, num_gaussians=1,
                                 not_terminal_loss_weight=200.0, seed=1)),
    # MDNRNNTrainerParameters() defaults over 6 steps, with terminal rows
    ("mdnrnn_defaults_seq", dict(S=5, A=2, T=6, B=256, discrete=True, p_terminal=0.2, seed=2)),
    # loss on the last step only, continuous action, odd sizes
    ("mdnrnn_fit_last_odd", dict(S=3, A=1, T=4, B=97, discrete=False, hidden_size=37,
                                 num_hidden_layers=3, num_gaussians=3,
                                 fit_only_one_next_step=True, seed=3)),
]


def main(only=None):
    for name, kw in CASES:
        if only and name not in only:
            continue
        trainer_case(name, **kw)
    if not only or "memory_input_maker" in only:
        input_maker_case()


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
