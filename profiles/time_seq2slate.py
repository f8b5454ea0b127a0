"""Time Seq2SlateTransformerNet's fused forward and rank against the same computations in eager
torch on the same GPU: the reference's modules (nn.TransformerEncoder, TransformerDecoderLayers
and the last layer's head-averaged cross-attention weights, pytorch_decoder_mask) run the
reference's way, including its rank loop that re-runs the decoder over the whole prefix at
every step.

Shapes (seeded, untrained networks):
  * tsp:  the reference's simple-TSP tests, B 4096, N 6, candidate dim 2, state dim 1,
          state_embed_dim 1, d 32, 2 heads, FFN 32, 2 layers, T 6;
  * wide: B 1024, N 32, state / candidate dims 64, d 128, 8 heads, FFN 512, 2 layers, T 10.
Alternating fused and eager in one process, medians over repetitions of back-to-back calls
between CUDA events (no_grad):
  * log_prob:     PER_SEQ_LOG_PROB_MODE (encoder + teacher-forced decoder);
  * greedy_rank:  RANK_MODE greedy;
  * sampled_rank: RANK_MODE sampling (fused: inverse CDF on torch.rand; eager: multinomial);
  * kernels:      each C entry point alone on arguments built once (no Python per call).
Each fused mode is one kernel launch.  The card's name, power limit and maximum SM clock are
read in the same run.

    python profiles/time_seq2slate.py --out DIR [--reps 5] [--steps 20]

Writes DIR/time_seq2slate_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import alternate, card_info, cuda_device, launch_us, write_result  # noqa: E402

SHAPES = {
    "tsp": dict(B=4096, N=6, C=2, S=1, se=1, d=32, H=2, F=32, L=2, T=6),
    "wide": dict(B=1024, N=32, C=64, S=64, se=None, d=128, H=8, F=512, L=2, T=10),
}


class Eager(object):
    """The reference's Seq2SlateTransformerModel forward in torch, on a copy of the fused net's
    parameters."""

    def __init__(self, net):
        import copy

        self.m = copy.deepcopy(net.seq2slate)
        self.m.eval()
        self.H = net.num_heads

    def encode(self, state, src):
        import math

        import torch

        m = self.m
        B, N, _ = src.shape
        ce = m.candidate_embedder.linear(src) * math.sqrt(m.candidate_embedder.dim_out)
        se = m.state_embedder.linear(state) * math.sqrt(m.state_embedder.dim_out)
        se = se.repeat(1, N).reshape(B, N, -1)
        x = torch.cat((se, ce), dim=2)
        return m.encoder.transformer_encoder(x.transpose(0, 1)).transpose(0, 1)

    def decode(self, memory, state, tgt_in_idx, tgt_in_seq):
        import math

        import torch

        m = self.m
        B, N, _ = memory.shape
        T = tgt_in_idx.shape[1]
        dev = memory.device
        ce = m.candidate_embedder.linear(tgt_in_seq) * math.sqrt(m.candidate_embedder.dim_out)
        se = m.state_embedder.linear(state) * math.sqrt(m.state_embedder.dim_out)
        se = se.repeat(1, T).reshape(B, T, -1)
        x = torch.cat((se, ce), dim=2)
        pos = torch.arange(0, T, device=dev).unsqueeze(0).repeat(B, 1).reshape(B, T, 1)
        x = torch.relu(m.positional_encoding_decoder.pos_embed(torch.cat((x, pos), dim=2)))
        # pytorch_decoder_mask
        mask_idx = torch.tril(tgt_in_idx.repeat(1, T).reshape(B, T, T), diagonal=0)
        src_mask = torch.zeros(B, T, N + 2, dtype=torch.bool, device=dev).scatter(2, mask_idx, 1)
        src_mask = src_mask[:, :, 2:].repeat_interleave(self.H, dim=0)
        tgt_mask = torch.triu(torch.ones(1, T, T, dtype=torch.bool, device=dev), 1).repeat(
            B * self.H, 1, 1)
        out, mem = x.transpose(0, 1), memory.transpose(0, 1)
        layers = m.decoder.layers
        for layer in layers[:-1]:
            out = layer(out, mem, tgt_mask=tgt_mask, memory_mask=src_mask)
        last = layers[-1]
        out = last.norm1(out + last.self_attn(out, out, out, attn_mask=tgt_mask)[0])
        _, w = last.multihead_attn(out, mem, mem, attn_mask=src_mask)
        return torch.cat((torch.zeros(B, T, 2, device=dev), w), dim=2)

    def log_prob(self, state, src, tgt_in_idx, tgt_in_seq, tgt_out_idx):
        import torch

        p = self.decode(self.encode(state, src), state, tgt_in_idx, tgt_in_seq)
        g = torch.gather(p, 2, tgt_out_idx.unsqueeze(2)).squeeze(2).prod(1, keepdim=True)
        return torch.log(g.clamp(min=1e-40))

    def rank(self, state, src, T, greedy):
        import torch

        memory = self.encode(state, src)
        B, N, C = src.shape
        dev = src.device
        feats = torch.zeros(B, N + 2, C, device=dev)
        feats[:, 2:] = src
        rows = torch.arange(B, device=dev).unsqueeze(1)
        tin = torch.full((B, 1), 1, dtype=torch.long, device=dev)
        probs = torch.zeros(B, T, N + 2, device=dev)
        for step in torch.arange(T, device=dev):
            p = self.decode(memory, state, tin, feats[rows, tin])[:, -1, :]
            nxt = (torch.max(p, dim=1)[1] if greedy
                   else torch.multinomial(p, num_samples=1, replacement=False)).reshape(B, 1)
            probs[:, step, :] = p
            tin = torch.cat([tin, nxt], dim=1)
        idx = tin[:, 1:]
        seq = torch.gather(probs, 2, idx.unsqueeze(2)).squeeze(2).prod(1, keepdim=True)
        return idx, probs, seq.clamp(min=1e-40)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory of the JSON result")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    dev = cuda_device(__file__)

    import torch

    from reagent_b200.core.types import PreprocessedRankingInput
    from reagent_b200.models import Seq2SlateMode, Seq2SlateOutputArch, Seq2SlateTransformerNet

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {"card": card_info(), "shapes": SHAPES, "unit": "us", "reps": args.reps,
           "steps": args.steps}
    n = args.steps

    def timed(fn):
        def run(_name, _rep):
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            return launch_us(fn, n, warmup=0)
        return run

    for name, c in SHAPES.items():
        torch.manual_seed(0)
        net = Seq2SlateTransformerNet(
            state_dim=c["S"], candidate_dim=c["C"], num_stacked_layers=c["L"], dim_model=c["d"],
            max_src_seq_len=c["N"], max_tgt_seq_len=c["T"],
            output_arch=Seq2SlateOutputArch.AUTOREGRESSIVE, temperature=1.0, num_heads=c["H"],
            dim_feedforward=c["F"], state_embed_dim=c["se"]).to(dev)
        eg = Eager(net)
        B, N, T = c["B"], c["N"], c["T"]
        state, src = torch.randn(B, c["S"], device=dev), torch.randn(B, N, c["C"], device=dev)
        action = torch.stack([torch.randperm(N)[:T] for _ in range(B)]).to(dev)
        inp = PreprocessedRankingInput.from_input(state=state, candidates=src, device=dev,
                                                  action=action)
        tin, tout, tseq = inp.tgt_in_idx, inp.tgt_out_idx, inp.tgt_in_seq.float_features
        r = res[name] = {}
        with torch.no_grad():
            # the two agree before anything is timed
            lf = net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE).log_probs
            le = eg.log_prob(state, src, tin, tseq, tout)
            r["log_prob_max_abs_diff"] = float((lf - le).abs().max())
            gf = net.rank(state, src, T, greedy=True).ranked_tgt_out_idx
            ge = eg.rank(state, src, T, greedy=True)[0]
            r["greedy_rank_rows_equal"] = float((gf == ge).all(1).float().mean())
            r["log_prob"] = alternate(["fused", "eager"], args.reps, lambda k, rep: timed(
                (lambda: net(inp, Seq2SlateMode.PER_SEQ_LOG_PROB_MODE)) if k == "fused"
                else (lambda: eg.log_prob(state, src, tin, tseq, tout)))(k, rep))
            for mode, greedy in (("greedy_rank", True), ("sampled_rank", False)):
                r[mode] = alternate(["fused", "eager"], args.reps, lambda k, rep: timed(
                    (lambda: net.rank(state, src, T, greedy=greedy)) if k == "fused"
                    else (lambda: eg.rank(state, src, T, greedy)))(k, rep))
            r["kernels"] = kernels_alone(net, state, src, tin, tout, tseq, T, args.reps, n)
    write_result(args.out, __file__, res)


def kernels_alone(net, state, src, tin, tout, tseq, T, reps, n):
    """Each C entry point alone, on arguments built once: the log-prob forward (per-sequence
    output), the greedy rank and the sampled rank, back-to-back launches between CUDA events."""
    import torch

    from profiles.timing import summary
    from reagent_b200 import _lib

    lib, st = _lib.lib(), _lib.cur_stream()
    B, N = src.shape[0], src.shape[1]
    dev = state.device
    seq = torch.empty(B, 1, device=dev)
    idx = torch.empty(B, T, dtype=torch.int64, device=dev)
    probs = torch.empty(B, T, N + 2, device=dev)
    rseq = torch.empty(B, 1, device=dev)
    noise = torch.rand(B, T, device=dev)
    fwd, keep_f = net._args(state, src, T, _lib.SEQ2SLATE_DECODE_FORCED)
    fwd.tgt_in_idx, fwd.tgt_out_idx, fwd.tgt_in_seq = tin.data_ptr(), tout.data_ptr(), tseq.data_ptr()
    fwd.seq_log_prob = seq.data_ptr()
    calls = {"rb200_seq2slate_forward": (lib.rb200_seq2slate_forward, fwd)}
    keep = [keep_f]
    for name, decode in (("rb200_seq2slate_rank_greedy", _lib.SEQ2SLATE_DECODE_GREEDY),
                         ("rb200_seq2slate_rank_sample", _lib.SEQ2SLATE_DECODE_SAMPLE)):
        a, k = net._args(state, src, T, decode)
        a.ranked_idx, a.probs, a.seq_prob = idx.data_ptr(), probs.data_ptr(), rseq.data_ptr()
        a.noise = noise.data_ptr()
        keep.append(k)
        calls[name] = (lib.rb200_seq2slate_rank, a)
    out = {}
    for name, (fn, a) in calls.items():
        def call(fn=fn, a=a, name=name):
            _lib.check(fn(a, st), name)
        out[name] = summary([launch_us(call, n, warmup=2) for _ in range(reps)])
    return out


if __name__ == "__main__":
    main()
