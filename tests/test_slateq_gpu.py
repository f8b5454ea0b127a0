"""SlateQ on the GPU: rb200_slateq_head against the float64 oracle (oracle/slateq_oracle.py) at
the edges of what it accepts, its limits and out-of-range indices; SlateQTrainer against the
goldens of the unmodified reference (oracle/make_slateq_golden.py); the input maker, scorer and
top-k sampler against theirs."""
import math
import random

import numpy as np
import pytest
import torch

from oracle import slateq_oracle as SO
from tests import golden_util as G
from tests import slateq_cases as SC

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _inputs(B, C, K, slate_size, *, maxq, Kn=None, seed=0, p_term=0.2, partial=True,
            time_diff=False):
    g = torch.Generator().manual_seed(seed)
    Kn = K if Kn is None else Kn
    d = dict(q_cur=torch.randn(B, K, generator=g), q_next=torch.randn(B, C, generator=g),
             next_value=torch.randn(B, C, generator=g),
             next_mask=(torch.rand(B, C, generator=g) > (0.3 if partial else -1)).float(),
             cur_mask=(torch.rand(B, C, generator=g) > (0.3 if partial else -1)).float(),
             next_action=None if maxq else torch.randint(0, C, (B, Kn), generator=g),
             action=torch.randint(0, C, (B, K), generator=g),
             reward=torch.randn(B, K, generator=g),
             reward_mask=(torch.rand(B, K, generator=g) > 0.5).float(),
             not_terminal=(torch.rand(B, generator=g) >= p_term).float(),
             time_diff=torch.randint(1, 5, (B,), generator=g).float() if time_diff else None)
    return d


def _head(d, *, gamma=0.9, slate_size, maxq, single, norm_next, time_scale=None, C=None):
    """One rb200_slateq_head call; returns (rc, outputs as CPU tensors)."""
    from reagent_b200 import _lib

    B, K = d["q_cur"].shape
    C = d["q_next"].shape[1] if C is None else C
    dv = {k: (None if v is None else v.to(DEV).contiguous()) for k, v in d.items()}
    out = dict(dz=torch.full((B * K,), 7.0, device=DEV), target=torch.empty(B * K, device=DEV),
               loss=torch.zeros(1, device=DEV), status=torch.zeros(1, dtype=torch.int32, device=DEV),
               count=torch.zeros(1, dtype=torch.int32, device=DEV),
               partials=torch.zeros((B + 7) // 8, device=DEV),
               counter=torch.zeros(1, dtype=torch.int32, device=DEV))
    a = _lib.SlateqArgsT()
    a.batch, a.num_candidates, a.slate_width = B, C, K
    a.next_width = 0 if dv["next_action"] is None else dv["next_action"].shape[1]
    a.slate_size, a.maxq, a.single_selection = slate_size, int(maxq), int(single)
    a.norm_method = _lib.SLATEQ_NORM_NEXT if norm_next else _lib.SLATEQ_NORM_CURRENT
    for k in ("q_cur", "q_next", "next_value", "next_mask", "cur_mask", "next_action", "action",
              "reward", "reward_mask", "not_terminal", "time_diff"):
        setattr(a, k, _lib.ptr(dv[k]))
    a.gamma = gamma
    a.time_scale = 0.0 if time_scale is None else time_scale
    a.dz, a.target, a.loss = out["dz"].data_ptr(), out["target"].data_ptr(), out["loss"].data_ptr()
    a.mask_count, a.status = out["count"].data_ptr(), out["status"].data_ptr()
    a.loss_partials, a.tile_counter = out["partials"].data_ptr(), out["counter"].data_ptr()
    rc = _lib.lib().rb200_slateq_head(a, _lib.cur_stream())
    torch.cuda.synchronize()
    res = {k: v.cpu() for k, v in out.items()}
    res["next_action"] = None if dv["next_action"] is None else dv["next_action"].cpu()
    return rc, res


def _check_against_oracle(d, *, slate_size, maxq, single, norm_next, gamma=0.9, time_scale=None):
    rc, got = _head(d, gamma=gamma, slate_size=slate_size, maxq=maxq, single=single,
                    norm_next=norm_next, time_scale=time_scale)
    assert rc == 0
    assert int(got["status"]) == 0
    target, nxt = SO.head_target(d["q_next"], d["next_value"], d["next_mask"], d["cur_mask"],
                                 d["next_action"], d["reward"], d["not_terminal"], d["time_diff"],
                                 gamma=gamma, slate_size=slate_size, maxq=maxq,
                                 single_selection=single, norm_next=norm_next,
                                 time_scale=time_scale)
    q = d["q_cur"].double().requires_grad_(True)
    loss = SO.head_loss(q, target, d["reward_mask"], single)
    (dz,) = torch.autograd.grad(loss, q)
    loss = loss.detach()
    B, K = d["q_cur"].shape
    # a row whose normalising mask is empty divides by 0 in the reference too: inf / NaN
    assert torch.allclose(got["target"].double().view(B, K), target, rtol=1e-5, atol=1e-5,
                          equal_nan=True)
    want, have = float(loss), float(got["loss"])
    if math.isnan(want):
        assert math.isnan(have)
    else:
        assert have == want or abs(have - want) <= 1e-5 * max(1.0, abs(want))
    assert torch.allclose(got["dz"].double().view(B, K), dz, rtol=1e-5, atol=1e-7, equal_nan=True)
    if not maxq:
        assert torch.equal(got["next_action"], nxt)
    return got


@pytest.mark.parametrize("maxq", [False, True])
@pytest.mark.parametrize("single,norm_next", [(True, False), (False, False), (False, True)])
@pytest.mark.parametrize("B,C,K,slate_size", [(1024, 10, 4, 3), (37, 7, 3, 2), (61, 100, 11, 10),
                                              (9, 5, 1, 5), (300, 4, 32, 4)])
def test_head_matches_the_oracle(maxq, single, norm_next, B, C, K, slate_size):
    """SARSA and top-k; single and multi selection; both normalisations; terminal rows;
    slate_size == C; K == 1 and K at its limit; B not a multiple of the block."""
    d = _inputs(B, C, K, slate_size, maxq=maxq, seed=B + C + K)
    _check_against_oracle(d, slate_size=slate_size, maxq=maxq, single=single, norm_next=norm_next)


def test_head_edges_time_diff_null_slot_and_duplicates():
    B, C, slate = 40, 10, 3
    d = _inputs(B, C, slate + 1, slate, maxq=False, seed=3, time_diff=True)
    # the null index (slate) also chosen in the slate; rows whose only reward is the null slot
    d["next_action"][:, -1] = slate
    d["next_action"][::3, 0] = slate
    d["reward_mask"][:, :-1] = 0.0
    d["reward_mask"][::2, -1] = 1.0
    d["not_terminal"][:5] = 0.0
    _check_against_oracle(d, slate_size=slate, maxq=False, single=True, norm_next=False,
                          gamma=0.95, time_scale=2.0)
    _check_against_oracle(d, slate_size=slate, maxq=True, single=False, norm_next=True,
                          time_scale=3.0)


def test_head_empty_reward_mask_gives_nan():
    d = _inputs(16, 6, 3, 2, maxq=False, seed=4)
    d["reward_mask"][:] = 0.0
    got = _check_against_oracle(d, slate_size=2, maxq=False, single=True, norm_next=False)
    assert (got["dz"] == 0).all() and int(got["count"]) == 0


def test_head_zeroes_terminal_next_actions_in_place():
    d = _inputs(50, 8, 3, 2, maxq=False, seed=5, p_term=0.5)
    _, got = _head(d, slate_size=2, maxq=False, single=True, norm_next=False)
    term = d["not_terminal"] == 0
    assert term.any()
    assert (got["next_action"][term] == 0).all()
    assert torch.equal(got["next_action"][~term], d["next_action"][~term])


def test_head_is_repeatable_bit_for_bit():
    d = _inputs(4096, 100, 11, 10, maxq=True, seed=6)
    runs = [_head(d, slate_size=10, maxq=True, single=True, norm_next=False)[1] for _ in range(3)]
    for r in runs[1:]:
        for k in ("dz", "target", "loss"):
            assert torch.equal(r[k].view(torch.int32), runs[0][k].view(torch.int32)), k


def test_head_reports_an_out_of_range_index():
    """An index of C in row 0 (its C-th element is still inside the allocation, so even a
    wrong kernel reads valid memory) is an IndexError in the reference; a negative index
    in [-C, 0) wraps as torch's indexing does."""
    B, C = 8, 6
    d = _inputs(B, C, 3, 2, maxq=False, seed=7, p_term=0.0)
    d["next_action"][0, 1] = C
    rc, got = _head(d, slate_size=2, maxq=False, single=True, norm_next=False)
    assert rc == 0 and int(got["status"]) == 1
    d = _inputs(B, C, 3, 2, maxq=True, seed=7, p_term=0.0)
    d["action"][0, 0] = C
    rc, got = _head(d, slate_size=2, maxq=True, single=True, norm_next=False)
    assert rc == 0 and int(got["status"]) == 1
    d = _inputs(B, C, 3, 2, maxq=False, seed=8, p_term=0.0)
    d["next_action"][1, 0] = -1
    got = _check_against_oracle(d, slate_size=2, maxq=False, single=True, norm_next=False)
    assert int(got["status"]) == 0


def test_head_limits():
    from reagent_b200 import _lib

    MC, MS = _lib.SLATEQ_MAX_CANDIDATES, _lib.SLATEQ_MAX_SLATE
    # at the limits
    d = _inputs(5, MC, MS, MS, maxq=True, seed=9)
    _check_against_oracle(d, slate_size=MS, maxq=True, single=True, norm_next=False)
    # just past them: C, K, K_next, slate_size > C
    for C, K, Kn, slate, maxq in [(MC + 1, 4, 4, 3, True), (40, MS + 1, 4, 3, True),
                                  (40, 4, MS + 1, 3, False), (5, 4, 4, 6, True),
                                  (40, 4, 4, MS + 1, True)]:
        d = _inputs(3, C, K, min(slate, C), maxq=maxq, Kn=Kn, seed=10)
        rc, _ = _head(d, slate_size=slate, maxq=maxq, single=True, norm_next=False)
        assert rc == _lib.E_INVALID, (C, K, Kn, slate)


# ---------------------------------------------------------------------------
# SlateQTrainer against the reference's goldens
# ---------------------------------------------------------------------------
def _trainer_from_golden(name):
    from reagent_b200.core.parameters import RLParameters, SlateOptMethod, SlateOptParameters
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import SlateQTrainer

    arrays, meta = G.load(name)
    q = FullyConnectedCritic(meta["S"], meta["D"], meta["sizes"], meta["acts"])
    G.load_into_module(arrays, "q0", q)
    q = q.cuda()
    qt = q.get_target_network()
    t = SlateQTrainer(
        q, qt, meta["slate_size"],
        rl=RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                        maxq_learning=meta["maxq"]),
        optimizer=Optimizer__Union.default(lr=meta["lr"]),
        slate_opt_parameters=(SlateOptParameters(method=SlateOptMethod.TOP_K)
                              if meta["maxq"] else None),
        discount_time_scale=meta["time_scale"], single_selection=meta["single_selection"],
        next_slate_value_norm_method=meta["norm"]).cuda()
    return t, arrays, meta


@pytest.mark.parametrize("name", SC.TRAINER_CASES)
@pytest.mark.parametrize("path", ["train_batch", "train_step_gen"])
def test_trainer_matches_the_goldens(name, path):
    from reagent_b200.core import types as rlt
    from reagent_b200.training import run_update

    t, arrays, meta = _trainer_from_golden(name)
    for it in range(meta["n_updates"]):
        batch = SC.slateq_input(SC.batch(arrays, it, DEV), rlt)
        if path == "train_batch":
            loss = float(t.train_batch(batch, it))
        else:
            loss = float(run_update(t, batch, it)[0])
        want = arrays["losses"][it]
        assert abs(loss - want) <= G.TOL * max(1.0, abs(want)), (it, loss, want)
        if not meta["maxq"]:
            assert np.array_equal(batch.next_action.cpu().numpy(),
                                  arrays[f"batch{it}.next_action_after"]), it
        else:
            assert np.array_equal(batch.next_action.cpu().numpy(), arrays[f"batch{it}.next_action"])
    t.raise_if_failed()
    G._cmp_module(t.q_network, arrays, "qN")
    G._cmp_module(t.q_network_target, arrays, "qtN")


def test_trainer_raises_index_error_for_an_out_of_range_slate():
    from reagent_b200.core import types as rlt

    t, arrays, meta = _trainer_from_golden("slateq_recsim_online")
    b = SC.batch(arrays, 0, DEV)
    b["next_action"][b["not_terminal"].view(-1).nonzero()[0, 0], 0] = meta["C"]
    t.train_batch(SC.slateq_input(b, rlt))
    with pytest.raises(IndexError):
        t.raise_if_failed()
    t.raise_if_failed()  # reported once


def test_maxq_recsim_yaml_without_slate_opt_parameters_raises():
    from reagent_b200.core import types as rlt
    m = SC.recsim_manager("slate_q_recsim_online_maxq_topk.yaml")
    t = m.build_trainer(SC.norm_map(20, 20), use_gpu=True)
    arrays, _ = G.load("slateq_recsim_online_maxq_topk")
    with pytest.raises(AssertionError):
        t.train_batch(SC.slateq_input(SC.batch(arrays, 0, DEV), rlt))


@pytest.mark.parametrize("yaml_name", sorted(SC.RECSIM_YAML.values()))
def test_manager_builds_and_trains_each_recsim_configuration(yaml_name):
    from dataclasses import replace

    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import SlateOptParameters
    from reagent_b200.optimizer import FusedAdam, SoftUpdate
    from reagent_b200.training import SlateQTrainer
    m = SC.recsim_manager(yaml_name)
    if m.trainer_param.rl.maxq_learning:
        m.trainer_param = replace(m.trainer_param, slate_opt_parameters=SlateOptParameters())
    torch.manual_seed(0)
    t = m.build_trainer(SC.norm_map(20, 20), use_gpu=True)
    assert isinstance(t, SlateQTrainer)
    assert [type(o["optimizer"]) for o in t.configure_optimizers()] == [FusedAdam, SoftUpdate]
    arrays, _ = G.load("slateq_recsim_online")
    for it in range(2):
        loss = float(t.train_batch(SC.slateq_input(SC.batch(arrays, it, DEV), rlt)))
        assert np.isfinite(loss)
    t.raise_if_failed()
    policy = m.create_policy(t)
    b = SC.batch(arrays, 0, DEV)
    obs = rlt.FeatureData(b["state"], candidate_docs=rlt.DocList(b["docs"], value=b["value"]))
    act = policy.act(obs)
    assert act.action.shape == (b["state"].shape[0], 3)


# ---------------------------------------------------------------------------
# input maker, scorer, sampler
# ---------------------------------------------------------------------------
def test_input_maker_matches_the_golden():
    from reagent_b200.gym.preprocessors.trainer_preprocessor import SlateQInputMaker
    from reagent_b200.replay_memory import ReplayBuffer

    arrays, meta = G.load("inputmaker_slateq")
    rb = ReplayBuffer(stack_size=1, replay_capacity=meta["cap"], batch_size=meta["B"])
    for t in range(meta["n_add"]):
        kw = {}
        for k in meta["keys"]:
            v = arrays[f"stream.{k}"][t]
            if k == "terminal":
                v = bool(v)
            elif np.ndim(v) == 0:
                v = float(v)
            kw[k] = v
        rb.add(**kw)
    maker = SlateQInputMaker()
    seed = meta["seed"] + 200
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    for s_i in range(meta["n_samples"]):
        raw = rb.sample_transition_batch(batch_size=meta["B"])
        out = maker(raw)
        pre = f"sample{s_i}."
        assert np.array_equal(raw.indices.cpu().numpy(), arrays[pre + "indices"])
        got = dict(state=out.state.float_features, next_state=out.next_state.float_features,
                   docs=out.state.candidate_docs.float_features,
                   next_docs=out.next_state.candidate_docs.float_features,
                   mask=out.state.candidate_docs.mask, next_mask=out.next_state.candidate_docs.mask,
                   value=out.state.candidate_docs.value,
                   next_value=out.next_state.candidate_docs.value, action=out.action,
                   next_action=out.next_action, reward=out.reward, reward_mask=out.reward_mask,
                   not_terminal=out.not_terminal)
        for k, v in got.items():
            want = arrays[pre + k]
            v = v.cpu().numpy()
            assert v.dtype == want.dtype and v.shape == want.shape, k
            assert np.array_equal(v, want), k


def test_scorer_and_top_k_sampler_match_the_golden():
    from reagent_b200.core import types as rlt
    from reagent_b200.gym.policies import TopKSampler, slate_q_scorer
    from reagent_b200.models import FullyConnectedCritic

    arrays, meta = G.load("slateq_scorer")
    q = FullyConnectedCritic(meta["S"], meta["D"], meta["sizes"], meta["acts"])
    G.load_into_module(arrays, "q", q)
    q = q.cuda()
    state = rlt.FeatureData(torch.from_numpy(arrays["obs"]).to(DEV),
                            candidate_docs=rlt.DocList(torch.from_numpy(arrays["docs"]).to(DEV),
                                                       value=torch.from_numpy(arrays["value"]).to(DEV)))
    scores = slate_q_scorer(meta["C"], q)(state)
    assert q.training
    assert G.rel_err(scores, arrays["scores"]) < G.TOL
    out = TopKSampler(k=meta["slate_size"]).sample_action(scores)
    assert np.array_equal(out.action.cpu().numpy(), arrays["action"])
    assert np.array_equal(out.log_prob.cpu().numpy(), arrays["log_prob"])
