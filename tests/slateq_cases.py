"""The SlateQ goldens (oracle/make_slateq_golden.py) and how the tests read them."""
import torch

from tests import golden_util as G

TRAINER_CASES = ["slateq_recsim_online", "slateq_recsim_online_with_time_scale",
                 "slateq_recsim_online_multi_selection",
                 "slateq_recsim_online_multi_selection_avg_curr", "slateq_recsim_online_maxq_topk",
                 "slateq_topk_multi", "slateq_time_diff", "slateq_odd_shapes"]

# the reference configuration each RecSim golden follows (gym/tests/configs/recsim/)
RECSIM_YAML = {"slateq_recsim_online": "slate_q_recsim_online.yaml",
               "slateq_recsim_online_with_time_scale": "slate_q_recsim_online_with_time_scale.yaml",
               "slateq_recsim_online_multi_selection": "slate_q_recsim_online_multi_selection.yaml",
               "slateq_recsim_online_multi_selection_avg_curr":
                   "slate_q_recsim_online_multi_selection_avg_curr.yaml",
               "slateq_recsim_online_maxq_topk": "slate_q_recsim_online_maxq_topk.yaml"}

BATCH_KEYS = ["state", "docs", "mask", "value", "next_state", "next_docs", "next_mask",
              "next_value", "action", "next_action", "reward", "reward_mask", "not_terminal",
              "time_diff"]


def batch(arrays, it, device="cpu"):
    """Update `it`'s batch as tensors (float16-stored values back to float32)."""
    out = {}
    for k in BATCH_KEYS:
        a = arrays.get(f"batch{it}.{k}")
        if a is None:
            out[k] = None
            continue
        t = torch.from_numpy(a.copy())
        out[k] = (t.float() if t.dtype == torch.float16 else t).to(device)
    return out


def oracle_kwargs(meta):
    return dict(gamma=meta["gamma"], slate_size=meta["slate_size"], maxq=meta["maxq"],
                single_selection=meta["single_selection"],
                norm_next=meta["norm"] == "norm_by_next_slate_size", time_scale=meta["time_scale"])


def oracle_nets(arrays, meta):
    from oracle.slateq_oracle import to64

    acts = meta["acts"] + ["linear"]
    return (to64(G.oracle_net(arrays, "q0", acts), requires_grad=True),
            to64(G.oracle_net(arrays, "qt0", acts)))


def slateq_input(b, rlt):
    """A reagent_b200 SlateQInput of a batch() dict."""
    def fd(s, d, m, v):
        return rlt.FeatureData(float_features=s, candidate_docs=rlt.DocList(d, m, v))

    return rlt.SlateQInput(
        state=fd(b["state"], b["docs"], b["mask"], b["value"]),
        next_state=fd(b["next_state"], b["next_docs"], b["next_mask"], b["next_value"]),
        reward=b["reward"], time_diff=b["time_diff"], step=None, not_terminal=b["not_terminal"],
        action=b["action"], next_action=b["next_action"], reward_mask=b["reward_mask"])


def recsim_manager(yaml_name):
    """The SlateQ manager with the fields of gym/tests/configs/recsim/<yaml_name>."""
    from reagent_b200.core.parameters import RLParameters, SlateQTrainerParameters
    from reagent_b200.model_managers import SlateQ
    from reagent_b200.net_builder import ParametricFullyConnected
    from reagent_b200.optimizer import Optimizer__Union

    tp = {}
    if yaml_name.endswith("_maxq_topk.yaml"):
        tp["rl"] = RLParameters(maxq_learning=True)
    if yaml_name.endswith("_with_time_scale.yaml"):
        tp["discount_time_scale"] = 2
    if "_multi_selection" in yaml_name:
        tp["single_selection"] = False
        tp["next_slate_value_norm_method"] = ("norm_by_current_slate_size"
                                              if yaml_name.endswith("_avg_curr.yaml")
                                              else "norm_by_next_slate_size")
    return SlateQ(slate_size=3, num_candidates=10, slate_feature_id=1, slate_score_id=(42, 42),
                  trainer_param=SlateQTrainerParameters(
                      optimizer=Optimizer__Union.default(lr=0.001), **tp),
                  net_builder=ParametricFullyConnected(sizes=[64, 64],
                                                       activations=["leaky_relu", "leaky_relu"]))


def norm_map(S, D):
    """STATE and ITEM normalizations of S and D continuous features."""
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters as NP

    return {"state": NormalizationData({i: NP("CONTINUOUS", mean=0.0, stddev=1.0) for i in range(S)}),
            "item": NormalizationData({100 + i: NP("CONTINUOUS", mean=0.0, stddev=1.0)
                                       for i in range(D)})}
