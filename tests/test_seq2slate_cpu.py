"""Seq2Slate without a GPU: the fp64 oracle against the reference's goldens, its sampled rank
against an independent restatement of the sample rule, the ranking input's index convention,
the shape limits, the workspace size and the net's parameter layout."""
import pytest
import torch

from oracle import seq2slate_oracle as O
from reagent_b200.core.types import PreprocessedRankingInput
from tests.seq2slate_cases import NAMES, load


@pytest.mark.parametrize("name", NAMES)
def test_oracle_log_probs_match_the_reference(name):
    meta, a, sd = load(name)
    sym, seq = O.log_probs(sd, _cfg(meta), a["state"], a["src_seq"], a["tgt_in_idx"],
                           a["tgt_in_seq"], a["tgt_out_idx"])
    torch.testing.assert_close(seq, a["log_prob.seq"].double(), rtol=1e-5, atol=1e-5)
    # log(1e-40) entries are exact; the rest are fp32 roundings of the fp64 values
    torch.testing.assert_close(sym, a["log_prob.symbol"].double(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_greedy_rank_matches_the_reference(name):
    meta, a, sd = load(name)
    idx, probs, seq = O.greedy_rank(sd, _cfg(meta), a["state"], a["src_seq"], meta["tgt_seq_len"])
    assert torch.equal(idx, a["rank.idx"])
    torch.testing.assert_close(probs, a["rank.symbol"].double(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(seq, a["rank.seq"].double(), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("name", NAMES)
def test_from_input_matches_the_reference(name):
    _, a, _ = load(name)
    inp = PreprocessedRankingInput.from_input(state=a["state"], candidates=a["src_seq"],
                                              device=torch.device("cpu"), action=a["action"])
    assert torch.equal(inp.tgt_in_idx, a["tgt_in_idx"])
    assert torch.equal(inp.tgt_out_idx, a["tgt_out_idx"])
    assert torch.equal(inp.tgt_in_seq.float_features, a["tgt_in_seq"])
    assert inp.tgt_in_idx[:, 0].eq(1).all() and inp.tgt_out_idx.min() >= 2
    assert inp.optim_tgt_out_idx is None and len(inp) == a["state"].shape[0]


def test_from_input_optimal_action():
    state, cands = torch.randn(3, 2), torch.randn(3, 4, 5)
    best = torch.tensor([[3, 0, 1], [1, 2, 0], [0, 1, 2]])
    inp = PreprocessedRankingInput.from_input(state=state, candidates=cands,
                                              device=torch.device("cpu"), optimal_action=best)
    assert inp.tgt_out_idx is None
    assert torch.equal(inp.optim_tgt_out_idx, best + 2)
    assert torch.equal(inp.optim_tgt_out_seq.float_features[1, 0], cands[1, 1])
    assert torch.equal(inp.optim_tgt_in_seq.float_features[:, 0], torch.zeros(3, 5))


def _net(**kw):
    from reagent_b200.models import Seq2SlateOutputArch, Seq2SlateTransformerNet

    args = dict(state_dim=3, candidate_dim=4, num_stacked_layers=2, dim_model=16,
                max_src_seq_len=6, max_tgt_seq_len=6,
                output_arch=Seq2SlateOutputArch.AUTOREGRESSIVE, temperature=1.0, num_heads=2,
                dim_feedforward=32)
    args.update(kw)
    return Seq2SlateTransformerNet(**args)


@pytest.mark.parametrize("kw", [
    dict(max_src_seq_len=65, max_tgt_seq_len=6),
    dict(max_tgt_seq_len=7),
    dict(dim_model=136, num_heads=2),
    dict(dim_model=18, num_heads=4),
    dict(dim_feedforward=513),
    dict(num_stacked_layers=5),
    dict(state_dim=257),
    dict(candidate_dim=257),
    dict(state_embed_dim=16),
])
def test_shape_limits_raise_value_error(kw):
    with pytest.raises(ValueError):
        _net(**kw)


def test_largest_shape_is_accepted():
    net = _net(max_src_seq_len=64, max_tgt_seq_len=64, dim_model=128, num_heads=2,
               dim_feedforward=512, num_stacked_layers=4, state_dim=256, candidate_dim=256)
    assert net.arena.flat.numel() == net.arena.n


def test_encoder_score_arch_is_not_implemented():
    from reagent_b200.models import Seq2SlateOutputArch

    with pytest.raises(NotImplementedError):
        _net(output_arch=Seq2SlateOutputArch.ENCODER_SCORE)


def test_parameters_are_views_of_one_arena_and_survive_deepcopy():
    import copy

    net = _net()
    flat = net.arena.flat
    for p in net.parameters():
        assert p.data.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
    clone = copy.deepcopy(net)
    assert clone.arena is not net.arena
    for (k, p), (k2, q) in zip(net.state_dict().items(), clone.state_dict().items()):
        assert k == k2 and torch.equal(p, q)
    for p in clone.parameters():
        assert p.data.untyped_storage().data_ptr() == clone.arena.flat.untyped_storage().data_ptr()


def test_slate_ranking_transformer_builds_the_net():
    from reagent_b200.core.parameters import TransformerParameters
    from reagent_b200.models import Seq2SlateOutputArch
    from reagent_b200.net_builder import SlateRankingTransformer

    b = SlateRankingTransformer()
    assert b.output_arch == Seq2SlateOutputArch.AUTOREGRESSIVE and b.temperature == 1.0
    assert b.transformer == TransformerParameters(num_heads=2, dim_model=16, dim_feedforward=16,
                                                  num_stacked_layers=2)
    b = SlateRankingTransformer(
        output_arch=Seq2SlateOutputArch.FRECHET_SORT, temperature=0.5,
        transformer=TransformerParameters(num_heads=3, dim_model=24, dim_feedforward=40,
                                          num_stacked_layers=3, state_embed_dim=5))
    torch.manual_seed(7)
    net = b.build_slate_ranking_network(state_dim=5, candidate_dim=3, candidate_size=7,
                                        slate_size=5)
    torch.manual_seed(7)
    direct = _net(state_dim=5, candidate_dim=3, num_stacked_layers=3, dim_model=24,
                  max_src_seq_len=7, max_tgt_seq_len=5,
                  output_arch=Seq2SlateOutputArch.FRECHET_SORT, temperature=0.5, num_heads=3,
                  dim_feedforward=40, state_embed_dim=5)
    assert (net.max_src_seq_len, net.max_tgt_seq_len, net.temperature) == (7, 5, 0.5)
    for (k, p), (k2, q) in zip(net.state_dict().items(), direct.state_dict().items()):
        assert k == k2 and torch.equal(p, q)
    assert net.seq2slate.state_embedder.linear.weight.shape == (5, 5)


def _cfg(meta):
    se = meta.get("state_embed_dim") or meta["dim_model"] // 2
    return dict(meta, state_embed_dim=se)


# ------------------------------------------------------------------------------------------
# The oracle's sampled rank, and the workspace size
# ------------------------------------------------------------------------------------------
# the largest fp32 uniform below 1, as the kernel reads it
ONE_BELOW = float(torch.nextafter(torch.tensor(1.0), torch.tensor(0.0)))


def _sampled(arch, noise_fn, N=7, T=7, B=5):
    """(state_dict, config, state, src_seq, noise, sample_rank's outputs) of a small net on the
    CPU."""
    from reagent_b200.models import Seq2SlateOutputArch

    torch.manual_seed(23)
    net = _net(max_src_seq_len=N, max_tgt_seq_len=T, output_arch=Seq2SlateOutputArch(arch))
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    cfg = dict(state_embed_dim=net.seq2slate.state_embed_dim, dim_model=16, num_stacked_layers=2,
               num_heads=2, output_arch=arch)
    g = torch.Generator().manual_seed(4)
    state, src = torch.randn(B, 3, generator=g), torch.randn(B, N, 4, generator=g)
    noise = noise_fn(B, T, g)
    return sd, cfg, state, src, noise, O.sample_rank(sd, cfg, state, src, T, noise)


ARCHS = ["autoregressive", "frechet_sort"]


@pytest.mark.parametrize("arch", ARCHS)
def test_sample_rank_is_the_inverse_cdf(arch):
    """Against torch.searchsorted: the first running sum strictly above u * total (such a
    symbol has nonzero probability), the last live symbol past the end."""
    _, _, _, _, noise, (idx, probs, seq, dist) = _sampled(
        arch, lambda B, T, g: torch.rand(B, T, generator=g))
    c = probs.cumsum(2)
    x = noise.double() * c[:, :, -1]
    j = torch.searchsorted(c, x.unsqueeze(2), right=True).squeeze(2)
    assert (j < probs.shape[2]).all()  # u < 1: some running sum exceeds u * total
    assert torch.equal(idx, j)
    assert (torch.gather(probs, 2, idx.unsqueeze(2)) > 0).all()
    assert all(len(set(r)) == len(r) for r in idx.tolist()) and idx.min() >= 2
    want = torch.gather(probs, 2, idx.unsqueeze(2)).squeeze(2).prod(1, keepdim=True)
    torch.testing.assert_close(seq, want.clamp(min=1e-40), rtol=0, atol=0)
    # the boundary distance is that of the nearest live running sum other than the total
    for b, t in [(0, 0), (1, 3), (4, 6)]:
        live = probs[b, t] > 0
        cb = c[b, t][live][:-1]
        want_d = (cb - x[b, t]).abs().min() if cb.numel() else torch.tensor(float("inf"))
        assert float(dist[b, t]) == float(want_d)


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("u", [0.0, ONE_BELOW, 1.0], ids=["zero", "one_below", "one"])
def test_sample_rank_edges_of_the_noise(arch, u):
    """u = 0 picks the first live symbol; nextafter(1, 0), and 1 itself (no running sum
    exceeds the total: the fallback), the last."""
    _, _, _, _, _, (idx, probs, _, dist) = _sampled(
        arch, lambda B, T, g: torch.full((B, T), u))
    live = probs > 0
    M = probs.shape[2]
    first = live.to(torch.int8).argmax(2)
    last = M - 1 - live.flip(2).to(torch.int8).argmax(2)
    assert torch.equal(idx, first if u == 0.0 else last)
    # the last step of a full-length rank has one live symbol and no boundary
    assert torch.equal(live[:, -1].sum(1), torch.ones(idx.shape[0], dtype=torch.long))
    assert torch.isinf(dist[:, -1]).all() and torch.isfinite(dist[:, :-1]).all()


def test_inverse_cdf_skips_zero_probabilities():
    p = torch.tensor([[0.0, 0.0, 0.25, 0.0, 0.5, 0.25, 0.0],
                      [0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0]], dtype=torch.float64)
    for u, want in [(0.0, 2), (0.24, 2), (0.25, 4), (0.74, 4), (0.75, 5), (0.99, 5), (1.0, 5)]:
        j, d = O.inverse_cdf(p, torch.tensor([u, u], dtype=torch.float64))
        assert j.tolist() == [want, 4]
        assert abs(float(d[0]) - min(abs(0.25 - u), abs(0.75 - u))) < 1e-15
        assert float(d[1]) == float("inf")


@pytest.mark.parametrize("arch", ARCHS)
def test_sample_rank_probs_are_the_decode_of_its_sequence(arch):
    sd, cfg, state, src, _, (idx, probs, _, _) = _sampled(
        arch, lambda B, T, g: torch.rand(B, T, generator=g))
    B = idx.shape[0]
    tin = torch.cat((torch.ones(B, 1, dtype=torch.long), idx[:, :-1]), dim=1)
    feats = torch.cat((torch.zeros(B, 2, src.shape[2]), src), dim=1)
    mem = O.encode(sd, cfg, state, src)
    ref = O.decode(sd, cfg, mem, state, tin, feats[torch.arange(B).unsqueeze(1), tin])
    torch.testing.assert_close(probs, ref, rtol=1e-12, atol=1e-15)


def test_greedy_top2_gap():
    sd, cfg, state, src, _, _ = _sampled("autoregressive", lambda B, T, g: torch.zeros(B, T))
    idx, probs, _ = O.greedy_rank(sd, cfg, state, src, 7)
    gap = O.top2_gap(probs)
    assert gap.shape == idx.shape and (gap >= 0).all()
    top = probs.sort(2, descending=True).values
    torch.testing.assert_close(gap, top[:, :, 0] - top[:, :, 1], rtol=0, atol=0)
    # the last step of a full-length rank: one live symbol against the zeros
    torch.testing.assert_close(gap[:, -1], torch.ones(idx.shape[0], dtype=torch.float64))


def _ws_args(B, N, T, C, d, H, F, L):
    from reagent_b200 import _lib

    a = _lib.Seq2slateArgsT()
    a.batch, a.src_len, a.tgt_len, a.state_dim, a.candidate_dim = B, N, T, 3, C
    a.state_embed_dim, a.dim_model, a.num_heads, a.dim_feedforward, a.layers = 1, d, H, F, L
    return a


def test_workspace_bytes_restatement():
    """The library's workspace size against tests/seq2slate_cases.ws_slice_bytes, on random
    shapes, the largest one and the two shapes at the shared / global boundary."""
    import random

    from reagent_b200 import _lib
    from tests.seq2slate_cases import (GLOBAL_EDGE, SMEM_EDGE, SMEM_MAX, workspace_bytes,
                                       ws_slice_bytes)

    assert ws_slice_bytes(**SMEM_EDGE) == SMEM_MAX
    assert ws_slice_bytes(**GLOBAL_EDGE) == SMEM_MAX + 16
    rng = random.Random(5)
    shapes = [SMEM_EDGE, GLOBAL_EDGE, dict(N=64, T=64, C=256, d=128, H=1, F=512, L=4)]
    for _ in range(300):
        d = rng.choice([2, 8, 16, 24, 32, 64, 96, 128])
        N = rng.randint(1, 64)
        shapes.append(dict(N=N, T=rng.randint(1, N), C=rng.randint(1, 256), d=d,
                           H=rng.choice([h for h in (1, 2, 4, 8, 16) if d % h == 0]),
                           F=rng.randint(1, 512), L=rng.randint(1, 4)))
    M = _lib.SEQ2SLATE_MAX_CTAS
    lib = _lib.lib()
    for s in shapes:
        for B in (1, 7, M - 1, M, M + 1, 2 * M + 1):
            got = lib.rb200_seq2slate_workspace_bytes(_ws_args(B, **s))
            assert got == workspace_bytes(B, M, **s), (s, B)
    assert lib.rb200_seq2slate_workspace_bytes(_ws_args(5, **SMEM_EDGE)) == 0
    assert lib.rb200_seq2slate_workspace_bytes(_ws_args(5, **GLOBAL_EDGE)) == 5 * (SMEM_MAX + 16)
