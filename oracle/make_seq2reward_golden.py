"""Generate the Seq2Reward golden vectors in tests/golden/ by running the UNMODIFIED reference
Seq2RewardTrainer, CompressModelTrainer and get_Q (reagent/training/world_model/
seq2reward_trainer.py, compress_model_trainer.py) through oracle/ref_harness.py.  Needs the
reference checkout (build container only); the files are committed.

    python oracle/make_seq2reward_golden.py            # regenerate every case
    python oracle/make_seq2reward_golden.py NAME ...   # only the named ones

The reference's model manager imports pyspark through WorldModelBase, so the networks are built
here the way its build_trainer builds them (Seq2RewardNetBuilder: Seq2RewardNetwork, then the
trainer builds its step network).  Shims on the trainer instance: `reporter` has no setter, so
`_reporter` is set to a recorder; configure_optimizers() returns dicts.

A trainer case holds
  p0.{i}.sha256 / sp0.{i}.sha256   SHA-256 of the seeded initial parameters of the Seq2Reward
                                   network / the step network, parameters() order
  batch{t}.{state,action,reward,valid_step}   the batch of update t
  out.acc_reward                   forward(state, action, valid_step) of batch 0, rows [0, 32)
  loss.mse / loss.step             get_mse_loss / get_step_entropy_loss of batch 0 under p0
  grad.{i} / sgrad.{i}             gradients of update 0 of both networks   } strided subsample
  p{t}.{i} / sp{t}.{i}             parameters after update t                } (SAMPLE_MAX)
  losses                           [update, (mse, step cross entropy)] as yielded
  val.{mse,step,q_values,action_distribution}   validation_step(batch 0) after the updates
  log.q_values                     the q_values the reporter logged each update (view_q_value)
A compress case holds the same for CompressModelTrainer (cp*, cgrad, losses [update], val.*,
`loss.{mse,accuracy}` before the updates, and `q` = get_Q of batch 0's first states).
A plan case holds `state`, `q` = get_Q at horizon k and `q_all` [B, k, A] = get_Q at every
horizon 1..k.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import _np, _save  # noqa: E402
from oracle.mdnrnn_oracle import digest, sample  # noqa: E402
from oracle.ref_harness import ref, run_update  # noqa: E402

OUT_ROWS = 32
N_UPDATES = 2


class Recorder:
    """A reporter that keeps what the trainer logs."""

    def __init__(self):
        self.logged = []

    def log(self, **kw):
        self.logged.append(kw)


def _batch(gen, S, A, T, B, k):
    action = torch.nn.functional.one_hot(torch.randint(A, (T, B), generator=gen), A).float()
    # valid steps spread over 1..min(T, k)
    valid = torch.arange(B) % min(T, k) + 1
    valid = valid[torch.randperm(B, generator=gen)]
    return dict(state=torch.randn(T, B, S, generator=gen), action=action,
                reward=torch.randn(T, B, generator=gen), valid_step=valid.unsqueeze(1))


def _input(b):
    rlt = ref("reagent.core.types")
    T, B = b["reward"].shape
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(float_features=b["state"]),
        next_state=rlt.FeatureData(float_features=b["state"]),
        action=rlt.FeatureData(float_features=b["action"]), reward=b["reward"],
        not_terminal=torch.ones(T, B), time_diff=None, step=None, valid_step=b["valid_step"])


def _params(**kw):
    return ref("reagent.core.parameters").Seq2RewardTrainerParameters(**kw)


def _network(S, A, H, L):
    return ref("reagent.models.seq2reward_model").Seq2RewardNetwork(
        state_dim=S, action_dim=A, num_hiddens=H, num_hidden_layers=L)


def trainer_case(name, *, S, A, T, B, H, L, k, seed=0, **param_kw):
    tm = ref("reagent.training.world_model.seq2reward_trainer")
    params = _params(multi_steps=k, action_names=[str(i) for i in range(A)], **param_kw)
    torch.manual_seed(seed)
    net = _network(S, A, H, L)
    trainer = tm.Seq2RewardTrainer(seq2reward_network=net, params=params)
    trainer._reporter = Recorder()
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    arrays = {}
    for i, p in enumerate(net.parameters()):
        arrays[f"p0.{i}.sha256"] = digest(p)
    for i, p in enumerate(trainer.step_predict_network.parameters()):
        arrays[f"sp0.{i}.sha256"] = digest(p)
    gen = torch.Generator().manual_seed(seed + 1000)
    batches = [_batch(gen, S, A, T, B, k) for _ in range(N_UPDATES)]
    for it, b in enumerate(batches):
        for key, v in b.items():
            arrays[f"batch{it}.{key}"] = _np(v).copy()
    b0 = _input(batches[0])
    with torch.no_grad():
        out = net(b0.state, b0.action, b0.valid_step.flatten()).acc_reward
        arrays["out.acc_reward"] = _np(out[:OUT_ROWS]).copy()
        arrays["loss.mse"] = np.array(float(trainer.get_mse_loss(b0)), dtype=np.float64)
        arrays["loss.step"] = np.array(float(trainer.get_step_entropy_loss(b0)), dtype=np.float64)
    losses = []
    for it, b in enumerate(batches):
        cap = {}
        losses.append(run_update(trainer, _input(b), it, opts, capture=cap))
        if it == 0:
            for i, g in enumerate(cap[0]):
                arrays[f"grad.{i}"] = _np(sample(g)).copy()
            for i, g in enumerate(cap[1]):
                arrays[f"sgrad.{i}"] = _np(sample(g)).copy()
        for i, p in enumerate(net.parameters()):
            arrays[f"p{it + 1}.{i}"] = _np(sample(p)).copy()
        for i, p in enumerate(trainer.step_predict_network.parameters()):
            arrays[f"sp{it + 1}.{i}"] = _np(sample(p)).copy()
    arrays["losses"] = np.array(losses, dtype=np.float64)
    arrays["log.q_values"] = np.array([r["q_values"][0] for r in trainer._reporter.logged
                                       if "q_values" in r], dtype=np.float64)
    mse, step, q_values, dist = trainer.validation_step(b0, 0)
    arrays["val.mse"] = np.array(mse, dtype=np.float64)
    arrays["val.step"] = np.array(step, dtype=np.float64)
    arrays["val.q_values"] = np.array(q_values, dtype=np.float64)
    arrays["val.action_distribution"] = np.array(dist, dtype=np.float64)
    _save(name, arrays, dict(kind="seq2reward", S=S, A=A, T=T, B=B, H=H, L=L, k=k, seed=seed,
                             lr=params.learning_rate, gamma=params.gamma,
                             view_q_value=params.view_q_value,
                             step_size=params.step_predict_net_size, n_updates=N_UPDATES))


def compress_case(name, *, S, A, T, B, H, L, k, sizes, seed=0, zero_head=False, **param_kw):
    cm = ref("reagent.training.world_model.compress_model_trainer")
    tm = ref("reagent.training.world_model.seq2reward_trainer")
    fc = ref("reagent.models.fully_connected_network")
    params = _params(multi_steps=k, action_names=[str(i) for i in range(A)], **param_kw)
    torch.manual_seed(seed)
    net = _network(S, A, H, L)
    comp = fc.FloatFeatureFullyConnected(state_dim=S, output_dim=A, sizes=sizes,
                                         activations=["relu"] * len(sizes))
    if zero_head:  # every sequence ties: pins the argmax rule of Q and of the accuracy
        with torch.no_grad():
            net.lstm_linear.weight.zero_()
    trainer = cm.CompressModelTrainer(compress_model_network=comp, seq2reward_network=net,
                                      params=params)
    trainer._reporter = Recorder()
    opts = [o["optimizer"] for o in trainer.configure_optimizers()]
    arrays = {}
    for i, p in enumerate(net.parameters()):
        arrays[f"p0.{i}.sha256"] = digest(p)
    for i, p in enumerate(comp.parameters()):
        arrays[f"cp0.{i}.sha256"] = digest(p)
    gen = torch.Generator().manual_seed(seed + 1000)
    batches = [_batch(gen, S, A, T, B, k) for _ in range(N_UPDATES)]
    for it, b in enumerate(batches):
        for key, v in b.items():
            arrays[f"batch{it}.{key}"] = _np(v).copy()
    b0 = _input(batches[0])
    with torch.no_grad():
        mse, acc = trainer.get_loss(b0)
        arrays["loss.mse"] = np.array(float(mse), dtype=np.float64)
        arrays["loss.accuracy"] = np.array(float(acc), dtype=np.float64)
        arrays["q"] = _np(tm.get_Q(net, b0.state.float_features[0], trainer.all_permut)).copy()
    losses = []
    for it, b in enumerate(batches):
        cap = {}
        losses.append(run_update(trainer, _input(b), it, opts, capture=cap)[0])
        if it == 0:
            for i, g in enumerate(cap[0]):
                arrays[f"cgrad.{i}"] = _np(sample(g)).copy()
        for i, p in enumerate(comp.parameters()):
            arrays[f"cp{it + 1}.{i}"] = _np(sample(p)).copy()
    arrays["losses"] = np.array(losses, dtype=np.float64)
    arrays["log.accuracy"] = np.array([r["accuracy"] for r in trainer._reporter.logged],
                                      dtype=np.float64)
    mse, q_values, dist, acc = trainer.validation_step(b0, 0)
    arrays["val.mse"] = np.array(mse, dtype=np.float64)
    arrays["val.q_values"] = np.array(q_values, dtype=np.float64)
    arrays["val.action_distribution"] = np.array(dist, dtype=np.float64)
    arrays["val.accuracy"] = np.array(acc, dtype=np.float64)
    _save(name, arrays, dict(kind="seq2reward_compress", S=S, A=A, T=T, B=B, H=H, L=L, k=k,
                             sizes=list(sizes), seed=seed, zero_head=zero_head,
                             lr=params.compress_model_learning_rate, n_updates=N_UPDATES))


def plan_case(name, *, S, A, k, B, H, L, seed=0):
    tm = ref("reagent.training.world_model.seq2reward_trainer")
    utils = ref("reagent.training.utils")
    torch.manual_seed(seed)
    net = _network(S, A, H, L)
    arrays = {f"p0.{i}.sha256": digest(p) for i, p in enumerate(net.parameters())}
    state = torch.randn(B, S, generator=torch.Generator().manual_seed(seed + 1000))
    arrays["state"] = _np(state).copy()
    q_all = torch.stack([tm.get_Q(net, state, utils.gen_permutations(j, A))
                         for j in range(1, k + 1)], dim=1)
    arrays["q"] = _np(tm.get_Q(net, state, utils.gen_permutations(k, A))).copy()
    arrays["q_all"] = _np(q_all).copy()
    arrays["permutations"] = _np(utils.gen_permutations(k, A)).copy()
    _save(name, arrays, dict(kind="seq2reward_plan", S=S, A=A, k=k, B=B, H=H, L=L, seed=seed))


TRAINER_CASES = [
    # seq2reward_test.yaml: Seq2RewardNetBuilder defaults, lr 0.005, multi_steps 6
    ("seq2reward_yaml", dict(S=2, A=2, T=6, B=1024, H=64, L=2, k=6, learning_rate=0.005)),
    ("seq2reward_odd", dict(S=5, A=3, T=4, B=37, H=37, L=1, k=4, gamma=0.9, view_q_value=True,
                            seed=1)),
    ("seq2reward_limits", dict(S=3, A=4, T=3, B=17, H=128, L=4, k=3, seed=2)),
]
COMPRESS_CASES = [
    ("seq2reward_compress", dict(S=2, A=2, T=6, B=256, H=64, L=2, k=6, sizes=[8, 8], seed=3)),
    ("seq2reward_compress_ties", dict(S=2, A=2, T=6, B=64, H=16, L=1, k=6, sizes=[8, 8], seed=4,
                                      zero_head=True)),
]
PLAN_CASES = [
    ("seq2reward_plan_a6_k1", dict(S=3, A=6, k=1, B=9, H=32, L=2, seed=5)),
    ("seq2reward_plan_a2_k3", dict(S=2, A=2, k=3, B=33, H=64, L=2, seed=6)),
    ("seq2reward_plan_a2_k6", dict(S=2, A=2, k=6, B=20, H=64, L=2, seed=7)),
    ("seq2reward_plan_a3_k4", dict(S=4, A=3, k=4, B=7, H=37, L=1, seed=8)),
]


def main(only=None):
    for cases, fn in ((TRAINER_CASES, trainer_case), (COMPRESS_CASES, compress_case),
                      (PLAN_CASES, plan_case)):
        for name, kw in cases:
            if not only or name in only:
                fn(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
