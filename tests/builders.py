"""Trainers and batches the GPU test modules share: DQNTrainer (with CPE heads or BCQ), QR-DQN,
SAC and TD3 from golden weights, their replay batches, the K2 kernel selection, and small
utilities of the GPU tests."""
import socket

import numpy as np
import torch

from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_util import TOL

# K2 has two implementations in the library: the warpgroup-MMA kernel (rb200_dqn_tc.cu,
# preferred when the shapes fit) and the mma.sync row-tile kernel (rb200_dqn.cu); every golden
# case runs on both.
K2_PATHS = ["wgmma", "rows"]


def _select_k2(monkeypatch, path):
    if path == "rows":
        monkeypatch.setenv("RB200_DISABLE_WGMMA", "1")
    else:
        monkeypatch.delenv("RB200_DISABLE_WGMMA", raising=False)


def _assert_k2(t, path):
    used_tc = t._last_td_call[-1] is not None
    assert used_tc == (path == "wgmma"), f"K2 ran on the wrong kernel (wanted {path})"


def _build_trainer(meta, arrays=None, dev="cuda"):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import DuelingQNetwork, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import DQNTrainer

    if meta.get("dueling"):
        q = DuelingQNetwork.make_fully_connected(meta["S"], meta["A"], meta["sizes"], meta["acts"])
    else:
        q = FullyConnectedDQN(meta["S"], meta["A"], meta["sizes"], meta["acts"])
    qt = q.get_target_network()
    if arrays is not None:
        G.load_into_module(arrays, "q0", q)
        G.load_into_module(arrays, "qt0", qt)
    q, qt = q.to(dev), qt.to(dev)
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                      q_network_loss=meta["loss"], maxq_learning=meta["maxq"],
                      multi_steps=meta["multi_steps"],
                      use_seq_num_diff_as_time_diff=meta["time_diff"],
                      reward_boost=meta["boost"])
    t = DQNTrainer(q, qt, actions=[str(i) for i in range(meta["A"])], rl=rl,
                   double_q_learning=meta["double_q"], minibatch_size=meta["B"],
                   optimizer=Optimizer__Union.default(lr=meta["lr"]),
                   evaluation=EvaluationParameters(calc_cpe_in_training=False))
    return t.to(dev)


def _rlt_batch(b, meta):
    from reagent_b200.core import types as rlt

    return rlt.DiscreteDqnInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
        reward=b["reward"], time_diff=b["time_diff"],
        step=b["step"] if meta["multi_steps"] is not None else None,
        not_terminal=b["not_terminal"], action=b["action"], next_action=b["next_action"],
        possible_actions_mask=b["possible_actions_mask"],
        possible_next_actions_mask=b["possible_next_actions_mask"],
        extras=rlt.ExtraData(action_probability=torch.ones_like(b["reward"])))


def _record(name, **kv):
    """Measurements the tolerances below are derived from, appended to
    $RB200_TEST_RECORD_DIR/test_measurements.jsonl when that variable names a directory."""
    import json, os
    d = os.environ.get("RB200_TEST_RECORD_DIR")
    if d and os.path.isdir(d):
        with open(os.path.join(d, "test_measurements.jsonl"), "a") as f:
            f.write(json.dumps({"test": name, **kv}) + "\n")


# Bounds of test_dqn_config2_matches_oracle: a hidden unit within ~5e-6 of 0 may take the other
# ReLU pattern than the oracle's, which moves its row's weight gradients; post-Adam elements
# within fp32 noise of a zero gradient move by +-lr.  Both are counted against these bounds.
CONFIG2_MAX_FLIPPED_ROWS = 8


CONFIG2_MAX_ADAM_OUTLIER_FRAC = 1.2e-3


# the mma.sync row-tile kernel (the library's second K2, taken when shapes do not fit the
# wgmma kernel) accumulates its 3xTF32 products in a different order, so per-row dZ gets 2e-5
CONFIG2_DZ_TOL = {"wgmma": TOL, "rows": 2e-5}


def _build_cpe_trainer(meta, arrays):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import DQNTrainer

    S, A = meta["S"], meta["A"]
    n_out = (len(meta["cpe_metrics"]) + 1) * A
    q = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"])
    qt = q.get_target_network()
    rn = FullyConnectedDQN(S, n_out, meta["sizes"], meta["acts"])
    qc = FullyConnectedDQN(S, n_out, meta["sizes"], meta["acts"])
    qct = qc.get_target_network()
    for net, prefix in ((q, "q0"), (qt, "qt0"), (rn, "r0"), (qc, "c0"), (qct, "ct0")):
        G.load_into_module(arrays, prefix, net)
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                      q_network_loss=meta["loss"], maxq_learning=meta["maxq"],
                      multi_steps=meta["multi_steps"], temperature=meta["temperature"],
                      use_seq_num_diff_as_time_diff=meta["time_diff"], reward_boost=meta["boost"])
    t = DQNTrainer(q.cuda(), qt.cuda(), rn.cuda(), qc.cuda(), qct.cuda(),
                   metrics_to_score=list(meta["cpe_metrics"]),
                   actions=[str(i) for i in range(A)], rl=rl, double_q_learning=meta["double_q"],
                   minibatch_size=meta["B"], optimizer=Optimizer__Union.default(lr=meta["lr"]),
                   evaluation=EvaluationParameters(calc_cpe_in_training=True))
    return t.cuda()


def _pbatch(b):
    from reagent_b200.core import types as rlt

    return rlt.PolicyNetworkInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
        action=rlt.FeatureData(b["action"]), next_action=rlt.FeatureData(b["next_action"]),
        reward=b["reward"], not_terminal=b["not_terminal"], step=None, time_diff=None,
        extras=rlt.ExtraData())


def _build_sac(meta, arrays):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import SACTrainer

    S, A = meta["S"], meta["A"]
    actor = GaussianFullyConnectedActor(S, A, meta["sizes"], meta["acts"])
    q1 = FullyConnectedCritic(S, A, meta["sizes"], meta["acts"])
    q2 = FullyConnectedCritic(S, A, meta["sizes"], meta["acts"]) if meta["twin"] else None
    G.load_into_module(arrays, "actor0", actor)
    G.load_into_module(arrays, "q1_0", q1)
    if q2 is not None:
        G.load_into_module(arrays, "q2_0", q2)
    opt = lambda: Optimizer__Union.default(lr=meta["lr"])  # noqa: E731
    kw = {} if meta["learn_alpha"] else {"alpha_optimizer": None}
    t = SACTrainer(actor, q1, q2, rl=RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"]),
                   q_network_optimizer=opt(), actor_network_optimizer=opt(),
                   minibatch_size=meta["B"], entropy_temperature=meta["entropy_temperature"],
                   target_entropy=meta["target_entropy"],
                   backprop_through_log_prob=meta["backprop"],
                   **({"alpha_optimizer": opt()} if meta["learn_alpha"] else kw))
    return t.cuda()


def _inject(t, arrays, it):
    def hook(name, shape, device):
        return torch.from_numpy(arrays[f"noise{it}.{name}"]).to(device)
    t.noise_hook = hook


def _build_td3(meta, arrays):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedActor, FullyConnectedCritic
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import TD3Trainer

    S, A = meta["S"], meta["A"]
    actor = FullyConnectedActor(S, A, meta["sizes"], meta["acts"])
    q1 = FullyConnectedCritic(S, A, meta["sizes"], meta["acts"])
    q2 = FullyConnectedCritic(S, A, meta["sizes"], meta["acts"]) if meta["twin"] else None
    G.load_into_module(arrays, "actor0", actor)
    G.load_into_module(arrays, "q1_0", q1)
    if q2 is not None:
        G.load_into_module(arrays, "q2_0", q2)
    opt = lambda: Optimizer__Union.default(lr=meta["lr"])  # noqa: E731
    t = TD3Trainer(actor, q1, q2, rl=RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"]),
                   q_network_optimizer=opt(), actor_network_optimizer=opt(),
                   minibatch_size=meta["B"], noise_variance=meta["noise_variance"],
                   noise_clip=meta["noise_clip"], delayed_policy_update=meta["delay"])
    return t.cuda()


def _rand_net(dims, acts, gen, bias=0.05):
    n = O.make_net(dims, acts, gen)
    for b in n["b"]:
        b.copy_(torch.randn(b.shape, generator=gen) * bias)
    return n


def _net_arrays(arrays, prefix, net):
    for i in range(len(net["W"])):
        arrays[f"{prefix}.W{i}"] = net["W"][i].detach().numpy().copy()
        arrays[f"{prefix}.b{i}"] = net["b"][i].detach().numpy().copy()


def _build_qr(meta, arrays):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import DuelingQNetwork, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import QRDQNTrainer

    if meta.get("dueling"):
        q = DuelingQNetwork.make_fully_connected(meta["S"], meta["A"], meta["sizes"], meta["acts"],
                                                 num_atoms=meta["N"])
    else:
        q = FullyConnectedDQN(meta["S"], meta["A"], meta["sizes"], meta["acts"], num_atoms=meta["N"])
    qt = q.get_target_network()
    G.load_into_module(arrays, "q0", q)
    G.load_into_module(arrays, "qt0", qt)
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                      maxq_learning=meta["maxq"], multi_steps=meta["multi_steps"])
    t = QRDQNTrainer(q, qt, actions=[str(i) for i in range(meta["A"])], rl=rl,
                     double_q_learning=meta["double_q"], num_atoms=meta["N"],
                     minibatch_size=meta["B"], optimizer=Optimizer__Union.default(lr=meta["lr"]),
                     evaluation=EvaluationParameters(calc_cpe_in_training=False))
    return t.cuda()


def _batch(b, meta):
    from reagent_b200.core import types as rlt

    return rlt.DiscreteDqnInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
        reward=b["reward"], time_diff=b["time_diff"],
        step=b["step"] if meta["multi_steps"] is not None else None,
        not_terminal=b["not_terminal"], action=b["action"], next_action=b["next_action"],
        possible_actions_mask=b["possible_actions_mask"],
        possible_next_actions_mask=b["possible_next_actions_mask"],
        extras=rlt.ExtraData())


def _build_bcq(meta, arrays=None, imitator=None, dev="cuda"):
    """DQNTrainer with BCQ (and CPE heads when meta["cpe_metrics"] is set) from golden weights."""
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import DuelingQNetwork, FullyConnectedDQN, FullyConnectedNetwork
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import DQNTrainer
    from reagent_b200.training.dqn_trainer import BCQConfig

    S, A = meta["S"], meta["A"]
    if meta.get("dueling"):
        q = DuelingQNetwork.make_fully_connected(S, A, meta["sizes"], meta["acts"])
    else:
        q = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"])
    qt = q.get_target_network()
    if imitator is None:
        imitator = FullyConnectedNetwork([S] + meta["imitator_sizes"] + [A], meta["imitator_acts"])
    nets, loads = (), [(q, "q0"), (qt, "qt0"), (imitator, "im")]
    cpe = meta.get("cpe_metrics") is not None
    if cpe:
        n_out = (len(meta["cpe_metrics"]) + 1) * A
        rn = FullyConnectedDQN(S, n_out, meta["sizes"], meta["acts"])
        qc = FullyConnectedDQN(S, n_out, meta["sizes"], meta["acts"])
        qct = qc.get_target_network()
        nets = (rn, qc, qct)
        loads += [(rn, "r0"), (qc, "c0"), (qct, "ct0")]
    if arrays is not None:
        for net, prefix in loads:
            G.load_into_module(arrays, prefix, net)
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                      q_network_loss=meta["loss"], maxq_learning=meta["maxq"],
                      multi_steps=meta["multi_steps"], temperature=meta.get("temperature", 0.01),
                      use_seq_num_diff_as_time_diff=meta["time_diff"], reward_boost=meta["boost"])
    t = DQNTrainer(q, qt, *nets, metrics_to_score=list(meta["cpe_metrics"]) if cpe else None,
                   actions=[str(i) for i in range(A)], rl=rl, double_q_learning=meta["double_q"],
                   minibatch_size=meta["B"], optimizer=Optimizer__Union.default(lr=meta["lr"]),
                   evaluation=EvaluationParameters(calc_cpe_in_training=cpe), imitator=imitator,
                   bcq=BCQConfig(meta["bcq"]))
    return t.to(dev)


def _golden_batch(arrays, meta):
    from reagent_b200.core import types as rlt

    b = G.batch_tensors(arrays, "cuda")
    batch = _rlt_batch(b, meta)
    batch.extras = rlt.ExtraData(action_probability=torch.ones_like(b["reward"]),
                                 metrics=b.get("metrics"))
    return b, batch


def _build_replay(arrays, meta, bulk=False):
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, ReplayBuffer

    if meta["prioritized"]:
        rb = PrioritizedReplayBuffer(stack_size=meta["stack"], replay_capacity=meta["cap"],
                                     batch_size=meta["B"], update_horizon=meta["horizon"],
                                     gamma=meta["gamma"])
    else:
        rb = ReplayBuffer(stack_size=meta["stack"], replay_capacity=meta["cap"],
                          batch_size=meta["B"], update_horizon=meta["horizon"],
                          gamma=meta["gamma"])
    keys = meta["keys"]
    st = {k: arrays[f"stream.{k}"] for k in keys}
    if bulk:
        rb.add_batch(**st)
        return rb
    for t in range(meta["n_add"]):
        kw = {}
        for k in keys:
            v = st[k][t]
            if k == "terminal":
                v = bool(v)
            elif k == "priority":
                v = float(v)
            elif k == "action" and not meta["continuous"]:
                v = int(v)
            elif np.ndim(v) == 0:
                v = float(v)
            kw[k] = v
        rb.add(**kw)
    return rb


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
