"""Seq2Slate without a GPU: the fp64 oracle against the reference's goldens, the ranking input's
index convention, the shape limits and the net's parameter layout."""
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
