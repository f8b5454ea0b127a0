"""Seq2SlateTransformerNet on the GPU: the fused forward and rank kernels against the reference's
goldens and the fp64 oracle, incremental decoding against a teacher-forced recompute, the
reference's propensity check, and sampling reproducibility."""
import itertools
import math

import pytest
import torch

from oracle import seq2slate_oracle as O
from reagent_b200.core.types import PreprocessedRankingInput
from reagent_b200.models import Seq2SlateMode, Seq2SlateOutputArch, Seq2SlateTransformerNet
from tests.seq2slate_cases import NAMES, build_net, load

pytestmark = pytest.mark.gpu


def _input(a, dev="cuda"):
    return PreprocessedRankingInput.from_input(state=a["state"], candidates=a["src_seq"],
                                               device=torch.device(dev), action=a["action"])


@pytest.mark.parametrize("name", NAMES)
def test_log_probs_match_the_reference(name):
    meta, a, sd = load(name)
    net = build_net(meta, sd)
    inp = _input(a)
    seq = net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs
    sym = net(inp, Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE).log_probs
    assert seq.shape == a["log_prob.seq"].shape and sym.shape == a["log_prob.symbol"].shape
    torch.testing.assert_close(seq.cpu(), a["log_prob.seq"], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(sym.cpu(), a["log_prob.symbol"], rtol=1e-5, atol=1e-5)
    # the symbols that can never be emitted keep the clamp's log of the fp32 denormal 1e-40
    # (no flush to zero), bit for bit
    assert torch.equal(sym[:, :, :2].cpu(), a["log_prob.symbol"][:, :, :2])


@pytest.mark.parametrize("name", NAMES)
def test_greedy_rank_matches_the_reference(name):
    meta, a, sd = load(name)
    net = build_net(meta, sd)
    out = net(_input(a), Seq2SlateMode.RANK_MODE, tgt_seq_len=meta["tgt_seq_len"], greedy=True)
    assert out.ranked_tgt_out_idx.dtype == torch.int64
    assert torch.equal(out.ranked_tgt_out_idx.cpu(), a["rank.idx"])
    torch.testing.assert_close(out.ranked_per_symbol_probs.cpu(), a["rank.symbol"], rtol=1e-5,
                               atol=1e-6)
    torch.testing.assert_close(out.ranked_per_seq_probs.cpu(), a["rank.seq"], rtol=1e-5,
                               atol=1e-7)


def _wide_net(arch, seed=0):
    torch.manual_seed(seed)
    return Seq2SlateTransformerNet(state_dim=64, candidate_dim=64, num_stacked_layers=2,
                                   dim_model=128, max_src_seq_len=32, max_tgt_seq_len=10,
                                   output_arch=arch, temperature=1.0, num_heads=8,
                                   dim_feedforward=512).cuda()


def _cfg(net):
    return dict(state_embed_dim=net.seq2slate.state_embed_dim, dim_model=net.dim_model,
                num_stacked_layers=net.num_stacked_layers, num_heads=net.num_heads,
                output_arch=net.output_arch.value)


@pytest.mark.parametrize("arch", [Seq2SlateOutputArch.AUTOREGRESSIVE,
                                  Seq2SlateOutputArch.FRECHET_SORT])
def test_wide_shape_against_the_fp64_oracle(arch):
    net = _wide_net(arch)
    B, N, T = 48, 32, 10
    g = torch.Generator().manual_seed(5)
    state, src = torch.randn(B, 64, generator=g), torch.randn(B, N, 64, generator=g)
    action = torch.stack([torch.randperm(N, generator=g)[:T] for _ in range(B)])
    inp = PreprocessedRankingInput.from_input(state=state, candidates=src,
                                              device=torch.device("cuda"), action=action)
    sym = net(inp, Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE).log_probs.cpu().double()
    seq = net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs.cpu().double()
    sd = {k: v.cpu() for k, v in net.state_dict().items()}
    osym, oseq = O.log_probs(sd, _cfg(net), state, src, inp.tgt_in_idx.cpu(),
                             inp.tgt_in_seq.float_features.cpu(), inp.tgt_out_idx.cpu())
    live = osym > math.log(1e-40)
    assert torch.equal(live, sym > math.log(1e-40))
    torch.testing.assert_close(sym[live], osym[live], rtol=1e-5, atol=2e-5)
    torch.testing.assert_close(seq, oseq, rtol=1e-5, atol=1e-4)


def test_largest_shape_runs_on_the_global_workspace():
    """N 64, d 128, FFN 512, 4 layers: a CTA's slice exceeds the shared-memory budget, so the
    kernel keeps it in the caller's workspace; same results as the fp64 oracle."""
    from reagent_b200 import _lib

    torch.manual_seed(3)
    net = Seq2SlateTransformerNet(state_dim=256, candidate_dim=256, num_stacked_layers=4,
                                  dim_model=128, max_src_seq_len=64, max_tgt_seq_len=64,
                                  output_arch=Seq2SlateOutputArch.AUTOREGRESSIVE,
                                  temperature=1.0, num_heads=2, dim_feedforward=512).cuda()
    B, N, T = 6, 64, 12
    state, src = torch.randn(B, 256), torch.randn(B, N, 256)
    action = torch.stack([torch.randperm(N)[:T] for _ in range(B)])
    inp = PreprocessedRankingInput.from_input(state=state, candidates=src,
                                              device=torch.device("cuda"), action=action)
    a, _ = net._args(inp.state.float_features, inp.src_seq.float_features, T,
                     _lib.SEQ2SLATE_DECODE_FORCED)
    assert a.workspace_bytes > 0
    sym = net(inp, Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE).log_probs.cpu().double()
    sd = {k: v.cpu() for k, v in net.state_dict().items()}
    osym, _ = O.log_probs(sd, _cfg(net), state, src, inp.tgt_in_idx.cpu(),
                          inp.tgt_in_seq.float_features.cpu(), inp.tgt_out_idx.cpu())
    live = osym > math.log(1e-40)
    torch.testing.assert_close(sym[live], osym[live], rtol=1e-5, atol=2e-5)
    out = net.rank(inp.state.float_features, inp.src_seq.float_features, T, greedy=True)
    _, oprobs, _ = O.greedy_rank(sd, _cfg(net), state, src, T)
    torch.testing.assert_close(out.ranked_per_symbol_probs.cpu().double(), oprobs, rtol=1e-4,
                               atol=1e-6)


@pytest.mark.parametrize("arch", [Seq2SlateOutputArch.AUTOREGRESSIVE,
                                  Seq2SlateOutputArch.FRECHET_SORT])
@pytest.mark.parametrize("greedy", [True, False])
def test_rank_probs_equal_a_teacher_forced_forward(arch, greedy):
    """The rank's per-step probabilities equal the teacher-forced forward on the sequence it
    ranked.  Both run the same incremental decoder, so this pins that the rank feeds it the
    symbols it chose; test_rank_probs_equal_a_full_recompute pins the decoder itself."""
    net = _wide_net(arch, seed=1)
    B, N, T = 64, 32, 10
    state, src = torch.randn(B, 64, device="cuda"), torch.randn(B, N, 64, device="cuda")
    out = net.rank(state, src, T, greedy=greedy)
    idx = out.ranked_tgt_out_idx
    assert idx.min() >= 2 and idx.max() < N + 2
    assert all(len(set(r)) == T for r in idx.tolist())  # a permutation prefix
    inp = PreprocessedRankingInput.from_input(state=state, candidates=src,
                                              device=torch.device("cuda"), action=idx - 2)
    fwd = net(inp, Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE).log_probs
    if arch == Seq2SlateOutputArch.FRECHET_SORT and greedy:
        # the argsort path: one-hot probabilities, and the ranking is by the first step's
        assert torch.equal(out.ranked_per_symbol_probs.sum(2), torch.ones(B, T, device="cuda"))
        first = fwd[:, 0].exp()
        assert (torch.gather(first, 1, idx).diff(dim=1) <= 0).all()
        return
    torch.testing.assert_close(out.ranked_per_symbol_probs.clamp(min=1e-40).log(), fwd,
                               rtol=1e-5, atol=1e-5)
    seq = net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs
    torch.testing.assert_close(out.ranked_per_seq_probs.log(), seq, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("arch", [Seq2SlateOutputArch.AUTOREGRESSIVE,
                                  Seq2SlateOutputArch.FRECHET_SORT])
@pytest.mark.parametrize("greedy", [True, False])
def test_rank_probs_equal_a_full_recompute(arch, greedy):
    """Incremental decoding (cached keys / values, one new row per step) against the fp64
    oracle's decoder, which recomputes every layer over the whole prefix as the reference's
    _autoregressive_rank does, on the sequence the kernel ranked."""
    net = _wide_net(arch, seed=4)
    B, N, T = 32, 32, 10
    state, src = torch.randn(B, 64), torch.randn(B, N, 64)
    out = net.rank(state.cuda(), src.cuda(), T, greedy=greedy)
    idx = out.ranked_tgt_out_idx.cpu()
    sd = {k: v.cpu() for k, v in net.state_dict().items()}
    cfg = _cfg(net)
    mem = O.encode(sd, cfg, state, src)
    tin = torch.cat((torch.ones(B, 1, dtype=torch.long), idx[:, :-1]), dim=1)
    feats = torch.cat((torch.zeros(B, 2, 64), src), dim=1)
    tseq = feats[torch.arange(B).unsqueeze(1), tin]
    ref = O.decode(sd, cfg, mem, state, tin, tseq)
    probs = out.ranked_per_symbol_probs.cpu().double()
    if arch == Seq2SlateOutputArch.FRECHET_SORT and greedy:
        # argsort of the first step's recomputed probabilities, one-hot outputs
        first = ref[:, 0].clone()
        first[:, :2] = -1.0
        want = torch.sort(first, dim=1, descending=True, stable=True).indices[:, :T]
        assert torch.equal(idx, want)
        return
    torch.testing.assert_close(probs, ref, rtol=1e-4, atol=1e-6)
    if greedy:
        assert torch.equal(idx, ref.argmax(2))


@pytest.mark.parametrize("arch", [Seq2SlateOutputArch.AUTOREGRESSIVE,
                                  Seq2SlateOutputArch.FRECHET_SORT])
def test_propensities_of_all_permutations(arch):
    """The reference's propensity check (test_seq2slate_inference / _propensity_computation):
    over the 24 permutations of 4 candidates the sequence probabilities sum to 1 and match the
    frequencies of sampled rankings."""
    torch.manual_seed(0)
    N = 4
    net = Seq2SlateTransformerNet(state_dim=2, candidate_dim=3, num_stacked_layers=2,
                                  dim_model=16, max_src_seq_len=N, max_tgt_seq_len=N,
                                  output_arch=arch, temperature=1.0, num_heads=2,
                                  dim_feedforward=32).cuda()
    state, src = torch.randn(1, 2, device="cuda"), torch.randn(1, N, 3, device="cuda")
    perms = torch.tensor(list(itertools.permutations(range(N))), device="cuda")
    P = perms.shape[0]
    inp = PreprocessedRankingInput.from_input(state=state.expand(P, 2),
                                              candidates=src.expand(P, N, 3),
                                              device=torch.device("cuda"), action=perms)
    probs = net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs.exp().reshape(-1)
    assert abs(float(probs.sum()) - 1.0) < 1e-5
    S = 200000
    out = net.rank(state.expand(S, 2), src.expand(S, N, 3), N, greedy=False)
    code = ((out.ranked_tgt_out_idx - 2) * torch.tensor([N ** 3, N ** 2, N, 1],
                                                        device="cuda")).sum(1)
    counts = torch.bincount(code, minlength=N ** 4)
    pcode = (perms * torch.tensor([N ** 3, N ** 2, N, 1], device="cuda")).sum(1)
    assert int(counts[pcode].sum()) == S  # only permutations are sampled
    freq = counts.float() / S
    assert float((freq[pcode] - probs).abs().max()) < 0.01
    # the reported per-seq probability of each sample is the one of its permutation
    lookup = torch.zeros(N ** 4, device="cuda")
    lookup[pcode] = probs
    torch.testing.assert_close(out.ranked_per_seq_probs.reshape(-1), lookup[code], rtol=1e-5,
                               atol=1e-6)


def test_sampled_rank_is_reproducible():
    net = _wide_net(Seq2SlateOutputArch.AUTOREGRESSIVE, seed=2)
    state, src = torch.randn(32, 64, device="cuda"), torch.randn(32, 32, 64, device="cuda")
    torch.manual_seed(11)
    a = net.rank(state, src, 10, greedy=False)
    torch.manual_seed(11)
    b = net.rank(state, src, 10, greedy=False)
    assert torch.equal(a.ranked_tgt_out_idx, b.ranked_tgt_out_idx)
    assert torch.equal(a.ranked_per_symbol_probs, b.ranked_per_symbol_probs)
    torch.manual_seed(11)
    noise = torch.rand(32, 10, device="cuda")
    c = net.rank(state, src, 10, greedy=False, noise=noise)
    assert torch.equal(a.ranked_tgt_out_idx, c.ranked_tgt_out_idx)
    # noise below every first cumulative probability picks the first live symbol
    z = net.rank(state, src, 10, greedy=False, noise=torch.zeros(32, 10, device="cuda"))
    first = (z.ranked_per_symbol_probs > 0).float().argmax(2)
    assert torch.equal(z.ranked_tgt_out_idx, first)


def test_modes_do_not_synchronise_with_the_host():
    meta, a, sd = load("seq2slate_tsp")
    net = build_net(meta, sd)
    inp = _input(a)
    noise = torch.rand(inp.batch_size(), meta["tgt_seq_len"], device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE)
        net(inp, Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE)
        net(inp, Seq2SlateMode.RANK_MODE, greedy=True)
        net(inp, Seq2SlateMode.RANK_MODE, greedy=False, noise=noise)
        net(inp, Seq2SlateMode.RANK_MODE, greedy=False)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_temperature_is_not_applied():
    meta, a, sd = load("seq2slate_autoregressive")
    hot = build_net(dict(meta, temperature=10.0), sd)
    cold = build_net(meta, sd)
    inp = _input(a)
    assert torch.equal(hot(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs,
                       cold(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs)


def test_host_tensors_are_refused():
    meta, a, sd = load("seq2slate_autoregressive")
    net = build_net(meta, sd)
    from reagent_b200 import _lib

    with pytest.raises(_lib.Rb200Error):
        net.rank(a["state"], a["src_seq"], 3, greedy=True)
    with pytest.raises(NotImplementedError):
        net(_input(a), Seq2SlateMode.ENCODER_SCORE_MODE)
