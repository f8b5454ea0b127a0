"""What the Seq2Reward tests share: the golden cases (oracle/make_seq2reward_golden.py), the
seeded networks they start from, checked against the goldens' SHA-256 digests, and the batches."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mdnrnn_oracle as mo  # noqa: E402

from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import (NormalizationData, NormalizationParameters,  # noqa: E402
                                          Seq2RewardTrainerParameters)
from reagent_b200.models import FloatFeatureFullyConnected, Seq2RewardNetwork  # noqa: E402
from reagent_b200.training import CompressModelTrainer, Seq2RewardTrainer  # noqa: E402

TRAINER_CASES = ["seq2reward_yaml", "seq2reward_odd", "seq2reward_limits"]
COMPRESS_CASES = ["seq2reward_compress", "seq2reward_compress_ties"]
PLAN_CASES = ["seq2reward_plan_a6_k1", "seq2reward_plan_a2_k3", "seq2reward_plan_a2_k6",
              "seq2reward_plan_a3_k4"]


class Recorder:
    """A reporter that keeps what the trainer logs."""

    def __init__(self):
        self.logged = []

    def log(self, **kw):
        self.logged.append(kw)


def check_digests(params, arrays, prefix):
    """The seeded parameters are the reference's, bit for bit."""
    params = list(params)
    assert len(params) == sum(k.startswith(prefix + "0.") for k in arrays)
    for i, p in enumerate(params):
        np.testing.assert_array_equal(mo.digest(p), arrays[f"{prefix}0.{i}.sha256"],
                                      err_msg=f"{prefix}0.{i}")


def norm(n):
    return NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS", mean=0.0, stddev=1.0)
        for i in range(n)})


def trainer_params(meta):
    return Seq2RewardTrainerParameters(
        learning_rate=meta["lr"], multi_steps=meta["k"],
        action_names=[str(i) for i in range(meta["A"])], gamma=meta["gamma"],
        view_q_value=meta["view_q_value"], step_predict_net_size=meta["step_size"])


def build_trainer(arrays, meta, device):
    """Seq2RewardTrainer as the golden built it under torch.manual_seed(seed)."""
    torch.manual_seed(meta["seed"])
    net = Seq2RewardNetwork(meta["S"], meta["A"], meta["H"], meta["L"])
    tr = Seq2RewardTrainer(net, trainer_params(meta)).to(device)
    check_digests(tr.seq2reward_network.parameters(), arrays, "p")
    check_digests(tr.step_predict_network.parameters(), arrays, "sp")
    return tr


def build_compress(arrays, meta, device):
    """(CompressModelTrainer, Seq2RewardNetwork) as the golden built them."""
    torch.manual_seed(meta["seed"])
    net = Seq2RewardNetwork(meta["S"], meta["A"], meta["H"], meta["L"])
    comp = FloatFeatureFullyConnected(meta["S"], meta["A"], meta["sizes"],
                                      ["relu"] * len(meta["sizes"]))
    if meta["zero_head"]:
        with torch.no_grad():
            net.lstm_linear.weight.zero_()
    net, comp = net.to(device), comp.to(device)
    check_digests(net.parameters(), arrays, "p")
    check_digests(comp.parameters(), arrays, "cp")
    params = Seq2RewardTrainerParameters(multi_steps=meta["k"],
                                         action_names=[str(i) for i in range(meta["A"])])
    return CompressModelTrainer(comp, net, params), net


def plan_network(arrays, meta, device):
    torch.manual_seed(meta["seed"])
    net = Seq2RewardNetwork(meta["S"], meta["A"], meta["H"], meta["L"]).to(device)
    check_digests(net.parameters(), arrays, "p")
    return net


def batch(arrays, it, device):
    g = lambda k: torch.from_numpy(arrays[f"batch{it}.{k}"]).to(device)  # noqa: E731
    T, B = arrays[f"batch{it}.reward"].shape
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(g("state")), next_state=rlt.FeatureData(g("state")),
        action=rlt.FeatureData(g("action")), reward=g("reward"),
        not_terminal=torch.ones(T, B, device=device), time_diff=None, step=None,
        valid_step=g("valid_step"))

