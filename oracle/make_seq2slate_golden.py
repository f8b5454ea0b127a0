"""Generate the Seq2Slate golden vectors in tests/golden/ by running the UNMODIFIED reference
Seq2SlateTransformerNet (reagent/models/seq2slate.py) through oracle/ref_harness.py.  Needs the
reference checkout (build container only); the files are committed.

    python oracle/make_seq2slate_golden.py            # regenerate every case
    python oracle/make_seq2slate_golden.py NAME ...   # only the named ones

The network is built under torch.manual_seed(seed) and the batch drawn after it.  A case holds
  p.<state_dict key>        the seeded initial parameters
  state, src_seq, action    the batch: action [B, T] is a random slate of distinct candidates
  tgt_in_idx, tgt_out_idx, tgt_in_seq    PreprocessedRankingInput.from_input(...) of it
  log_prob.seq              PER_SEQ_LOG_PROB_MODE [B, 1]
  log_prob.symbol           PER_SYMBOL_LOG_PROB_DIST_MODE [B, T, N + 2]
  rank.idx, rank.symbol, rank.seq        RANK_MODE greedy with tgt_seq_len T
and __meta__ the model's constructor arguments.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import _np, _save  # noqa: E402
from oracle.ref_harness import ref  # noqa: E402

# name: (constructor arguments, batch, tgt_seq_len, seed)
CASES = {
    "seq2slate_autoregressive": (dict(state_dim=3, candidate_dim=4, num_stacked_layers=2,
                                      dim_model=16, max_src_seq_len=6, max_tgt_seq_len=6,
                                      output_arch="autoregressive", temperature=1.0,
                                      num_heads=2, dim_feedforward=32), 32, 6, 0),
    "seq2slate_frechet_sort": (dict(state_dim=3, candidate_dim=4, num_stacked_layers=2,
                                    dim_model=16, max_src_seq_len=6, max_tgt_seq_len=6,
                                    output_arch="frechet_sort", temperature=1.0,
                                    num_heads=2, dim_feedforward=32), 32, 6, 1),
    # the reference's simple-TSP shape (test_seq2slate_on_policy / off_policy)
    "seq2slate_tsp": (dict(state_dim=1, candidate_dim=2, num_stacked_layers=2, dim_model=32,
                           max_src_seq_len=6, max_tgt_seq_len=6, output_arch="autoregressive",
                           temperature=1.0, num_heads=2, dim_feedforward=32, state_embed_dim=1),
                      64, 6, 2),
    # odd sizes: N 7, d 24 over 3 heads, FFN 40, 3 layers, T < N
    "seq2slate_odd": (dict(state_dim=5, candidate_dim=3, num_stacked_layers=3, dim_model=24,
                           max_src_seq_len=7, max_tgt_seq_len=5, output_arch="autoregressive",
                           temperature=0.5, num_heads=3, dim_feedforward=40, state_embed_dim=5),
                      24, 5, 3),
}


def make(name):
    cfg, B, T, seed = CASES[name]
    S = ref("reagent.models.seq2slate")
    U = ref("reagent.model_utils.seq2slate_utils")
    rlt = ref("reagent.core.types")
    torch.manual_seed(seed)
    kw = dict(cfg, output_arch=U.Seq2SlateOutputArch(cfg["output_arch"]))
    net = S.Seq2SlateTransformerNet(**kw).eval()
    N, C = cfg["max_src_seq_len"], cfg["candidate_dim"]
    state = torch.randn(B, cfg["state_dim"])
    src_seq = torch.randn(B, N, C)
    action = torch.stack([torch.randperm(N)[:T] for _ in range(B)])
    inp = rlt.PreprocessedRankingInput.from_input(state=state, candidates=src_seq,
                                                  device=torch.device("cpu"), action=action)
    arrays = {"p." + k: _np(v) for k, v in net.state_dict().items()}
    arrays.update(state=_np(state), src_seq=_np(src_seq), action=_np(action),
                  tgt_in_idx=_np(inp.tgt_in_idx), tgt_out_idx=_np(inp.tgt_out_idx),
                  tgt_in_seq=_np(inp.tgt_in_seq.float_features))
    with torch.no_grad():
        arrays["log_prob.seq"] = _np(net(inp, U.Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs)
        arrays["log_prob.symbol"] = _np(
            net(inp, U.Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE).log_probs)
        out = net(inp, U.Seq2SlateMode.RANK_MODE, tgt_seq_len=T, greedy=True)
    arrays["rank.idx"] = _np(out.ranked_tgt_out_idx)
    arrays["rank.symbol"] = _np(out.ranked_per_symbol_probs)
    arrays["rank.seq"] = _np(out.ranked_per_seq_probs)
    _save(name, arrays, dict(cfg, batch=B, tgt_seq_len=T, seed=seed))


def main(only=None):
    for name in CASES:
        if not only or name in only:
            make(name)


if __name__ == "__main__":
    main(sys.argv[1:])
