"""GPU parity: fused CUDA DQN update vs (a) golden vectors from the unmodified reference and
(b) the CPU oracle at BASELINE config-2 size.  Tolerance: 1e-5 relative fp32 (north star)."""
import numpy as np
import pytest
import torch

from oracle import td_oracle as O
from tests import golden_util as G
from tests.builders import (CONFIG2_DZ_TOL, CONFIG2_MAX_ADAM_OUTLIER_FRAC, CONFIG2_MAX_FLIPPED_ROWS,
                            K2_PATHS, _assert_k2, _build_cpe_trainer, _build_trainer, _record,
                            _rlt_batch, _select_k2)
from tests.golden_cases import DQN_CASES, DQN_CPE_CASES
from tests.golden_util import TOL

pytestmark = pytest.mark.gpu
# the BASELINE configs[0]-shaped case has 49 k hidden elements and 8.9 k parameters: it gets the
# size-aware post-Adam criterion of the config-2 test (test_dqn_config0_matches_reference)
CONFIG0 = "dqn_cartpole_config0"
DQN_CASES = [c for c in DQN_CASES if c != CONFIG0]


def _check_against_golden(t, arrays, meta, losses):
    for it, l in enumerate(losses):
        ref = arrays["losses"][it]
        assert abs(l - ref) <= TOL * max(1.0, abs(ref)), (it, l, ref)
    for net, prefix in ((t.q_network, "qN"), (t.q_network_target, "qtN")):
        ps = list(net.parameters())
        pairs = G.net_pairs(arrays, prefix)
        assert len(ps) == 2 * len(pairs)
        for i, (w, b) in enumerate(pairs):
            assert G.rel_err(ps[2 * i], w) < TOL, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], b) < TOL, (prefix, i)


@pytest.mark.parametrize("path", K2_PATHS)
@pytest.mark.parametrize("name", DQN_CASES)
def test_dqn_generator_path_matches_reference(name, path, monkeypatch):
    from reagent_b200.training import run_update

    _select_k2(monkeypatch, path)
    arrays, meta = G.load(name)
    t = _build_trainer(meta, arrays)
    batch = _rlt_batch(G.batch_tensors(arrays, "cuda"), meta)
    losses = []
    for it in range(meta["n_updates"]):
        gen_losses = None
        if it == 0:
            # drive the generator by hand once to inspect gradients before the Adam step
            opts = t.optimizers()
            loss = t.training_step(batch, it, 0)
            grads = t.q_network_grads()
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < TOL, f"grad {i}"
            assert G.rel_err(t.all_action_scores, arrays["all_q0"]) < TOL
            assert loss.grad_fn is not None
            opts[0].zero_grad(); loss.backward(); opts[0].step()
            l2 = t.training_step(batch, it, 1)
            opts[1].zero_grad(); l2.backward(); opts[1].step()
            losses.append(float(loss))
        else:
            gen_losses = run_update(t, batch, it)
            assert len(gen_losses) == 2
            losses.append(float(gen_losses[0]))
    _assert_k2(t, path)
    _check_against_golden(t, arrays, meta, losses)


@pytest.mark.parametrize("path", K2_PATHS)
@pytest.mark.parametrize("name", DQN_CASES)
def test_dqn_fast_path_matches_reference(name, path, monkeypatch):
    _select_k2(monkeypatch, path)
    arrays, meta = G.load(name)
    t = _build_trainer(meta, arrays)
    batch = _rlt_batch(G.batch_tensors(arrays, "cuda"), meta)
    losses = [float(t.train_batch(batch, it)) for it in range(meta["n_updates"])]
    _assert_k2(t, path)
    _check_against_golden(t, arrays, meta, losses)


@pytest.mark.parametrize("path", K2_PATHS)
def test_dqn_config2_matches_oracle(path, monkeypatch):
    """BASELINE config 2 shapes: S=128, A=16, B=4096, [256,128] relu, double-Q, huber.
    1e-5 (north star) on everything computed on rows whose activation pattern equals the
    oracle's; the number of other rows is asserted small; the weight gradient is compared at
    1e-5 with exactly those rows' contributions exchanged."""
    _select_k2(monkeypatch, path)
    meta = dict(S=128, A=16, B=4096, sizes=[256, 128], acts=["relu", "relu"], gamma=0.99,
                tau=0.005, loss="huber", maxq=True, multi_steps=None, time_diff=False,
                boost=None, double_q=True, lr=1e-3, n_updates=3)
    gen = torch.Generator().manual_seed(0)
    B, S, A = meta["B"], meta["S"], meta["A"]
    q = O.make_net([S, 256, 128, A], ["relu", "relu", "linear"], gen)
    qt = O.clone_net(q)
    for w in qt["W"]:
        w.add_(torch.randn(w.shape, generator=gen) * 0.02)
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = q["W"][i].numpy().copy(), q["b"][i].numpy().copy()
        arrays[f"qt0.W{i}"], arrays[f"qt0.b{i}"] = qt["W"][i].numpy().copy(), qt["b"][i].numpy().copy()
    act = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.005).float()
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen), time_diff=torch.ones(B, 1), step=None,
             not_terminal=nt, action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    t = _build_trainer(meta, arrays)
    qo = O.clone_net(q, requires_grad=True)
    adam = O.AdamState(O.net_params(qo), lr=meta["lr"])
    gb = {k: (v.cuda() if v is not None else None) for k, v in b.items()}
    batch = _rlt_batch(gb, meta)

    # ---- per-row view of the first update on the oracle side: z_l, h_l, dLoss/dz_l ----
    def oracle_rows():
        hs, zs = [], []
        x = b["state"]
        for w, bb, a in zip(qo["W"], qo["b"], qo["act"]):
            z = torch.nn.functional.linear(x, w, bb)
            z.retain_grad()
            zs.append(z)
            x = torch.relu(z) if a == "relu" else z
            hs.append(x)
        _, aux = O.dqn_td_loss(qo, qt, b, gamma=meta["gamma"], double_q=True, maxq=True, loss="huber")
        q_sel = torch.sum(hs[-1] * b["action"], 1, keepdim=True)
        loss = torch.nn.functional.smooth_l1_loss(q_sel, aux["target"])
        loss.backward()
        dz = [z.grad.detach().clone() for z in zs]
        for p_ in O.net_params(qo):
            p_.grad = None
        return [h.detach() for h in hs], dz

    h_ref, dz_ref = oracle_rows()
    flipped = None
    for it in range(meta["n_updates"]):
        lo, grads, aux = O.dqn_update(qo, qt, adam, b, gamma=meta["gamma"], tau=meta["tau"],
                                      double_q=True, maxq=True, loss="huber")
        t._td_step(batch)
        _assert_k2(t, path)
        if it == 0:
            assert torch.equal(t._ws["next_idx"].cpu().long(), aux["next_idx"].reshape(-1))
            assert G.rel_err(t._ws["td_target"], aux["target"].reshape(-1)) < TOL
            assert G.rel_err(t._ws["scores"], aux["all_q"]) < TOL
            net = t._ws["net"]
            h_gpu = [h.cpu() for h in net.hidden]
            dz_gpu = [z.cpu() for z in net.dz]
            same = torch.ones(B, dtype=torch.bool)
            for l in range(2):
                same &= ((h_gpu[l] > 0) == (h_ref[l] > 0)).all(dim=1)
            flipped = int((~same).sum())
            assert flipped <= CONFIG2_MAX_FLIPPED_ROWS, flipped
            for l in range(2):  # saved activations: 1e-5 everywhere (a flip moves h by < 1e-5)
                assert G.rel_err(h_gpu[l], h_ref[l]) < TOL, ("hidden", l)
            for l in range(3):  # dLoss/dz per row: 1e-5 on the rows with the oracle's pattern
                assert G.rel_err(dz_gpu[l][same], dz_ref[l][same]) < CONFIG2_DZ_TOL[path], ("dz", l)
            # weight gradients at 1e-5: the oracle's, with the flipped rows' contributions
            # replaced by what follows from the GPU's own dz on those rows
            inputs = [b["state"]] + h_ref[:2]
            g_gpu = t.q_network_grads()
            worst = 0.0
            for l in range(3):
                dzm = dz_ref[l].clone()
                dzm[~same] = dz_gpu[l][~same]
                gw = dzm.double().t() @ inputs[l].double()
                gb_ = dzm.double().sum(0)
                ew, eb = G.rel_err(g_gpu[2 * l], gw), G.rel_err(g_gpu[2 * l + 1], gb_)
                worst = max(worst, ew, eb)
                assert ew < CONFIG2_DZ_TOL[path] and eb < CONFIG2_DZ_TOL[path], ("wgrad", l, ew, eb)
            # and against the unmodified oracle gradient: bounded by the flipped rows' weight
            l2mx = [G.grad_close(g, grads[i], f"grad {i}", l2_tol=1e-4, max_tol=1e-4)
                    for i, g in enumerate(g_gpu)]
            _record("dqn_config2", path=path, flipped_rows=flipped, wgrad_rel_err_masked=worst,
                    grad_l2_rel=max(x[0] for x in l2mx), grad_max_rel=max(x[1] for x in l2mx))
        t.optimizers()[0].fused_step(target=t.q_network_target.arena, tau=t.tau)
        assert abs(float(t._ws["loss"]) - lo) <= 2e-5 * max(1.0, abs(lo))
    # post-Adam parameters: an element whose gradient is within fp32 noise of zero moves by
    # up to lr per step in either direction (Adam normalises the step), so every element is
    # bounded by the total step size and the fraction off by more than 1e-5 is bounded at 10x
    # the measured one
    fracs = []
    for i, seq in enumerate(t.q_network.fc.dnn):
        d = (seq[0].weight.detach().cpu().double() - qo["W"][i].detach().double()).abs()
        assert float(d.max()) <= 2.0 * meta["n_updates"] * meta["lr"] * 1.01
        fracs.append(float((d > 1e-5 * float(qo["W"][i].abs().max())).double().mean()))
    _record("dqn_config2_adam", path=path, outlier_frac=fracs)
    assert max(fracs) < CONFIG2_MAX_ADAM_OUTLIER_FRAC, fracs
    for i, seq in enumerate(t.q_network_target.fc.dnn):
        assert G.rel_err(seq[0].weight, qt["W"][i]) < TOL


def test_mlp_forward_matches_torch():
    from reagent_b200.core import types as rlt
    from reagent_b200.models import FullyConnectedCritic, FullyConnectedDQN

    torch.manual_seed(1)
    for (S, A, sizes, acts, B) in [(128, 16, [256, 128], ["relu", "relu"], 4096),
                                   (7, 3, [10, 6], ["tanh", "leaky_relu"], 37),
                                   (5, 2, [300], ["sigmoid"], 1)]:
        q = FullyConnectedDQN(S, A, sizes, acts)
        x = torch.randn(B, S)
        ref = x
        for seq in q.fc.dnn:
            ref = seq(ref)
        out = q.cuda()(rlt.FeatureData(x.cuda()))
        assert G.rel_err(out, ref) < TOL
    c = FullyConnectedCritic(256, 32, [256, 256], ["relu", "relu"])
    s, a = torch.randn(2048, 256), torch.rand(2048, 32) * 2 - 1
    ref = torch.cat([s, a], 1)
    for seq in c.fc.dnn:
        ref = seq(ref)
    out = c.cuda()(rlt.FeatureData(s.cuda()), rlt.FeatureData(a.cuda()))
    assert G.rel_err(out, ref) < TOL


@pytest.mark.parametrize("B,S,sizes,A,acts,loss,double_q,maxq", [
    (4096, 128, [256, 128], 16, ["relu", "relu"], "huber", True, True),   # BASELINE config 2
    (100, 10, [24, 12], 3, ["tanh", "relu"], "mse", False, True),         # ragged rows, odd dims
    (33, 7, [40], 5, ["leaky_relu"], "huber", True, False),               # SARSA, one hidden layer
    (257, 36, [300, 130, 20], 9, ["relu", "sigmoid", "relu"], "mse", True, True),  # >128-wide tiles
])
def test_k2_wgmma_matches_rows_kernel(B, S, sizes, A, acts, loss, double_q, maxq):
    """The two K2 kernels on identical inputs: every output (loss, scores, TD target, arg max,
    saved activations, dZ of every layer) within 1e-5 of the tensor's scale; arg max bit-exact."""
    from reagent_b200 import _lib

    meta = dict(S=S, A=A, B=B, sizes=sizes, acts=acts, gamma=0.97, tau=0.01, loss=loss,
                maxq=maxq, multi_steps=None, time_diff=False, boost=None, double_q=double_q,
                lr=1e-3, n_updates=1)
    torch.manual_seed(B + S)
    t = _build_trainer(meta)
    with torch.no_grad():
        for p_ in t.q_network_target.parameters():
            p_.add_(0.05 * torch.randn_like(p_))
    act = torch.randint(A, (B,))
    nact = torch.randint(A, (B,))
    nt = (torch.rand(B, 1) > 0.1).float()
    mask = (torch.rand(B, A) > 0.3).float()
    mask[torch.arange(B), nact] = 1.0
    b = dict(state=torch.randn(B, S), next_state=torch.randn(B, S), reward=torch.randn(B, 1),
             time_diff=torch.ones(B, 1), step=None, not_terminal=nt,
             action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(nact, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=mask)
    batch = _rlt_batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    t._td_step(batch)
    qd, qtd, a, wsc, keep, pack = t._last_td_call
    assert pack is not None, "shapes expected to fit the wgmma path"
    ws, st = t._ws, _lib.cur_stream()

    def run(tc):
        for x in ws["net"].hidden + ws["net"].dz:
            x.zero_()
        if tc:
            rc = _lib.lib().rb200_dqn_td_step_tc(qd, qtd, a, wsc, pack.data_ptr(), pack.numel(), 0, st)
        else:
            rc = _lib.lib().rb200_dqn_td_step(qd, qtd, a, wsc, st)
        _lib.check(rc, "k2")
        torch.cuda.synchronize()
        out = {"loss": ws["loss"].clone(), "scores": ws["scores"].clone(),
               "tgt": ws["td_target"].clone(), "qsel": ws["q_sel"].clone(), "idx": ws["next_idx"].clone()}
        out.update({f"h{i}": h.clone() for i, h in enumerate(ws["net"].hidden)})
        out.update({f"dz{i}": z.clone() for i, z in enumerate(ws["net"].dz)})
        return out

    r_rows, r_tc = run(False), run(True)
    assert torch.equal(r_rows["idx"], r_tc["idx"])
    # Batch rows on which both kernels took the same activation branches.  A hidden unit whose
    # pre-activation is within fp32 noise of 0 can get the other ReLU mask (see
    # golden_util.grad_close), which legitimately changes that row's dZ; such rows are rare
    # and are excluded from the element-wise dZ comparison.
    same = torch.ones(B, dtype=torch.bool, device="cuda")
    for i in range(len(sizes)):
        same &= ((r_rows[f"h{i}"] > 0) == (r_tc[f"h{i}"] > 0)).all(dim=1)
    assert float(same.float().mean()) > 0.99
    for k in r_rows:
        if k == "idx":
            continue
        x, y = r_rows[k].double(), r_tc[k].double()
        scale = max(float(x.abs().max()), 1e-30)
        if k.startswith("dz"):
            x, y = x[same], y[same]
        # two 3xTF32 kernels, each within 1e-5 of the fp32 answer: 2e-5 between them
        assert float((x - y).abs().max()) <= 2 * TOL * scale, (k, float((x - y).abs().max()), scale)


def test_dueling_forward_heads_and_state_dict():
    """DuelingQNetwork: the folded single-launch forward, the head-by-head evaluation on the
    true parameters and the reference's q(s) agree; state_dict keys are the reference's."""
    from reagent_b200.core import types as rlt
    from reagent_b200.models import DuelingQNetwork

    arrays, meta = G.load("dqn_dueling_double")
    q = DuelingQNetwork.make_fully_connected(meta["S"], meta["A"], meta["sizes"], meta["acts"])
    assert list(q.state_dict().keys())[:2] == ["shared_network.fc.dnn.0.0.weight",
                                               "shared_network.fc.dnn.0.0.bias"]
    assert "advantage_network.fc.dnn.1.0.weight" in q.state_dict()
    assert tuple(q.state_dict()["value_network.fc.dnn.1.0.weight"].shape) == (1, meta["sizes"][-1] // 2)
    G.load_into_module(arrays, "q0", q)
    q = q.cuda()
    x = rlt.FeatureData(torch.from_numpy(arrays["batch.state"]).cuda())
    out = q(x)
    assert G.rel_err(out, arrays["all_q0"]) < TOL
    value, raw_adv, adv, qv = q._get_values(x)
    assert value.shape == (meta["B"], 1) and raw_adv.shape == (meta["B"], meta["A"])
    assert G.rel_err(qv, arrays["all_q0"]) < TOL
    assert float(adv.mean(dim=1).abs().max()) < 1e-6
    mask = torch.ones(meta["B"], meta["A"], device="cuda")
    mask[:, 0] = 0
    assert float(q(x, mask)[:, 0].max()) < -1e9
    # a copy through state_dict (what loading a reference checkpoint does) reproduces q
    q2 = DuelingQNetwork.make_fully_connected(meta["S"], meta["A"], meta["sizes"], meta["acts"]).cuda()
    q2.load_state_dict(q.state_dict())
    assert torch.equal(q2(x), out)
    qt = q.get_target_network()
    assert torch.equal(qt(x), out)


@pytest.mark.parametrize("S,sizes,A", [(128, [256, 128], 16), (10, [24, 12], 3), (36, [300, 130, 20], 9),
                                     # the edges of the wgmma plan: K = 1 and 480, a one-row
                                     # last tile, a fourth tile, A over 128
                                     (1, [129], 7), (7, [400], 9), (480, [8], 4), (8, [8], 141)])
def test_adam_writes_the_same_weight_images_as_the_pack_kernel(S, sizes, A):
    """The fused Adam kernel writes the hi/lo tensor-core images of the updated parameters;
    they must be bit-identical to what rb200_dqn_tc_pack builds from the same parameters."""
    from reagent_b200 import _lib

    B = 64
    meta = dict(S=S, A=A, B=B, sizes=sizes, acts=["relu"] * len(sizes), gamma=0.9, tau=0.1,
                loss="huber", maxq=True, multi_steps=None, time_diff=False, boost=None,
                double_q=True, lr=1e-2, n_updates=1)
    torch.manual_seed(S)
    t = _build_trainer(meta)
    act = torch.randint(A, (B,))
    nt = (torch.rand(B, 1) > 0.1).float()
    b = dict(state=torch.randn(B, S), next_state=torch.randn(B, S), reward=torch.randn(B, 1),
             time_diff=torch.ones(B, 1), step=None, not_terminal=nt,
             action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    batch = _rlt_batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    for _ in range(2):
        t.train_batch(batch)
    assert t._tc_images_current(), "the Adam step should have refreshed the images"
    qd, qtd, a, wsc, keep, pack = t._last_td_call
    assert pack is not None
    torch.cuda.synchronize()
    by_adam = pack.clone()
    fresh = torch.zeros_like(pack)
    rc = _lib.lib().rb200_dqn_tc_pack(t.q_network.arena.desc(), t.q_network_target.arena.desc(), 1, 1,
                                      fresh.data_ptr(), fresh.numel(), _lib.cur_stream())
    _lib.check(rc, "rb200_dqn_tc_pack")
    torch.cuda.synchronize()
    assert torch.equal(by_adam, fresh)
    # an in-place torch write to the parameters (what load_state_dict does) invalidates them
    with torch.no_grad():
        next(t.q_network.parameters()).mul_(1.0)
    assert not t._tc_images_current()


@pytest.mark.parametrize("path", K2_PATHS)
def test_dqn_config0_matches_reference(path, monkeypatch):
    """BASELINE configs[0] shapes (the reference's own CPU-runnable DQN workflow: S=4, A=2, B=256,
    [128,64] leaky_relu, double-Q, mse, Adam 0.01, tau 0.2) against vectors from the unmodified
    reference: loss, q(s) and every gradient to 1e-5; post-Adam parameters with the step-size
    aware bound (an Adam step turns a gradient element that is within fp32 summation noise of
    zero into a move of up to lr, so elements are bounded by lr and all but a vanishing fraction
    must agree to 1e-5 -- same criterion as the config-2 test)."""
    _select_k2(monkeypatch, path)
    arrays, meta = G.load(CONFIG0)
    t = _build_trainer(meta, arrays)
    batch = _rlt_batch(G.batch_tensors(arrays, "cuda"), meta)
    assert meta["n_updates"] == 1
    t._td_step(batch)
    _assert_k2(t, path)
    ref_loss = float(arrays["losses"][0])
    assert abs(float(t._ws["loss"]) - ref_loss) <= TOL * max(1.0, abs(ref_loss))
    assert G.rel_err(t.all_action_scores, arrays["all_q0"]) < TOL
    for i, g in enumerate(t.q_network_grads()):
        assert G.rel_err(g, arrays[f"grad0.{i}"]) < TOL, f"grad {i}"
    t.optimizers()[0].fused_step(target=t.q_network_target.arena, tau=t.tau)
    for net, prefix in ((t.q_network, "qN"), (t.q_network_target, "qtN")):
        ps = list(net.parameters())
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            for got, ref in ((ps[2 * i], w), (ps[2 * i + 1], b)):
                d = (got.detach().cpu().double() - torch.from_numpy(ref).double()).abs()
                assert float(d.max()) <= 2.0 * meta["lr"] * 1.01, (prefix, i)
                frac = float((d > TOL * float(np.abs(ref).max())).double().mean())
                assert frac < 0.01, (prefix, i, frac)


# ---------------------------------------------------------------------------
# CPE heads (calc_cpe_in_training=True, the reference default): dqn_trainer_base.py:243-452
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("name", DQN_CPE_CASES)
def test_dqn_cpe_matches_reference(name, fast):
    from reagent_b200.core import types as rlt
    from reagent_b200.training import run_update
    from reagent_b200.training.workspace import param_grads

    arrays, meta = G.load(name)
    t = _build_cpe_trainer(meta, arrays)
    assert len(t.configure_optimizers()) == 4
    b = G.batch_tensors(arrays, "cuda")
    batch = _rlt_batch(b, meta)
    batch.extras = rlt.ExtraData(action_probability=torch.ones_like(b["reward"]),
                                 metrics=b.get("metrics"))
    for it in range(meta["n_updates"]):
        if fast:
            td = float(t.train_batch(batch, it))
            rl_, cl_ = (float(x) for x in t.cpe_losses)
        else:
            out = run_update(t, batch, it)
            assert len(out) == 4
            td, rl_, cl_ = float(out[0]), float(out[1]), float(out[2])
        for got, want in ((td, arrays["losses"][it]), (rl_, arrays["cpe_losses"][it][0]),
                          (cl_, arrays["cpe_losses"][it][1])):
            assert abs(got - want) <= TOL * max(1.0, abs(want)), (it, got, want)
    for net, prefix in ((t.q_network, "qN"), (t.q_network_target, "qtN"), (t.reward_network, "rN"),
                        (t.q_network_cpe, "cN"), (t.q_network_cpe_target, "ctN")):
        ps = list(net.parameters())
        for i, (w, bb) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < TOL, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], bb) < TOL, (prefix, i)


def test_dqn_cpe_gradients_match_reference():
    from reagent_b200.core import types as rlt
    from reagent_b200.training.workspace import param_grads

    arrays, meta = G.load("dqn_cpe_huber")
    t = _build_cpe_trainer(meta, arrays)
    b = G.batch_tensors(arrays, "cuda")
    batch = _rlt_batch(b, meta)
    batch.extras = rlt.ExtraData(action_probability=torch.ones_like(b["reward"]), metrics=b.get("metrics"))
    opts = t.optimizers()
    l0 = t.training_step(batch, 0, 0)
    opts[0].zero_grad(); l0.backward(); opts[0].step()
    l1 = t.training_step(batch, 0, 1)  # reward loss: both CPE gradients exist from here on
    for i, g in enumerate(param_grads(t.reward_network.arena, list(t.reward_network.parameters()))):
        assert G.rel_err(g, arrays[f"grad0r.{i}"]) < TOL, f"reward grad {i}"
    for i, g in enumerate(param_grads(t.q_network_cpe.arena, list(t.q_network_cpe.parameters()))):
        assert G.rel_err(g, arrays[f"grad0c.{i}"]) < TOL, f"cpe grad {i}"
    assert abs(float(l1) - arrays["cpe_losses"][0][0]) <= TOL * max(1.0, abs(arrays["cpe_losses"][0][0]))
