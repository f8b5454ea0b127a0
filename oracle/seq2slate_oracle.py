"""float64 restatement of the Seq2Slate transformer (reagent/models/seq2slate.py) from a
state_dict: the encoder, the teacher-forced decoder over the whole prefix (full recompute, as
the reference does it) and the greedy and sampled ranks that re-run that decoder at every
step.  It is
written from the math (post-norm layers, per-head softmax attention, the pytorch_decoder_mask
masks), not from torch's transformer modules, and pinned against the reference's goldens by
tests/test_seq2slate_cpu.py."""
import math

import torch

F64 = torch.float64


def _p(sd, k):
    return sd[k].to(F64)


def _ln(x, g, b):
    m = x.mean(-1, keepdim=True)
    v = ((x - m) ** 2).mean(-1, keepdim=True)
    return (x - m) / torch.sqrt(v + 1e-5) * g + b


def _mha(q_in, kv_in, w, b, heads, mask=None):
    """Per-head attention of q_in [B, Tq, d] over kv_in [B, Tk, d] with in_proj (w, b);
    mask [B, Tq, Tk] True = ignore.  Returns (concatenated heads [B, Tq, d], weights
    [B, H, Tq, Tk])."""
    d = q_in.shape[-1]
    hd = d // heads
    q = q_in @ w[:d].T + b[:d]
    k = kv_in @ w[d:2 * d].T + b[d:2 * d]
    v = kv_in @ w[2 * d:].T + b[2 * d:]
    B, Tq, Tk = q.shape[0], q.shape[1], k.shape[1]
    q = q.view(B, Tq, heads, hd).transpose(1, 2)
    k = k.view(B, Tk, heads, hd).transpose(1, 2)
    v = v.view(B, Tk, heads, hd).transpose(1, 2)
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    if mask is not None:
        s = s.masked_fill(mask.unsqueeze(1), float("-inf"))
    p = torch.softmax(s, -1)
    return (p @ v).transpose(1, 2).reshape(B, Tq, d), p


def encode(sd, cfg, state, src_seq):
    """memory [B, N, d] of state [B, S] and src_seq [B, N, C]."""
    pre = "seq2slate."
    se = cfg["state_embed_dim"]
    ce = cfg["dim_model"] - se
    B, N, _ = src_seq.shape
    st = (state.to(F64) @ _p(sd, pre + "state_embedder.linear.weight").T
          + _p(sd, pre + "state_embedder.linear.bias")) * math.sqrt(se)
    ca = (src_seq.to(F64) @ _p(sd, pre + "candidate_embedder.linear.weight").T
          + _p(sd, pre + "candidate_embedder.linear.bias")) * math.sqrt(ce)
    x = torch.cat((st.unsqueeze(1).expand(B, N, se), ca), dim=2)
    for l in range(cfg["num_stacked_layers"]):
        k = f"{pre}encoder.transformer_encoder.layers.{l}."
        a, _ = _mha(x, x, _p(sd, k + "self_attn.in_proj_weight"),
                    _p(sd, k + "self_attn.in_proj_bias"), cfg["num_heads"])
        a = a @ _p(sd, k + "self_attn.out_proj.weight").T + _p(sd, k + "self_attn.out_proj.bias")
        x = _ln(x + a, _p(sd, k + "norm1.weight"), _p(sd, k + "norm1.bias"))
        f = torch.relu(x @ _p(sd, k + "linear1.weight").T + _p(sd, k + "linear1.bias"))
        f = f @ _p(sd, k + "linear2.weight").T + _p(sd, k + "linear2.bias")
        x = _ln(x + f, _p(sd, k + "norm2.weight"), _p(sd, k + "norm2.bias"))
    return x


def _src_mask(tgt_in_idx, N):
    """[B, T, N] True where candidate j was an input at a position <= t."""
    B, T = tgt_in_idx.shape
    m = torch.zeros(B, T, N + 2, dtype=torch.bool)
    for t in range(T):
        m[:, t].scatter_(1, tgt_in_idx[:, : t + 1], True)
    return m[:, :, 2:]


def decode(sd, cfg, memory, state, tgt_in_idx, tgt_in_seq):
    """Per-symbol probabilities [B, T, N + 2] of the teacher-forced decoder."""
    pre = "seq2slate."
    B, N, d = memory.shape
    T = tgt_in_idx.shape[1]
    mask = _src_mask(tgt_in_idx, N)
    if cfg["output_arch"] == "frechet_sort":
        sc = (memory @ _p(sd, pre + "encoder_scorer.weight").T
              + _p(sd, pre + "encoder_scorer.bias")).squeeze(2)
        logits = sc.unsqueeze(1).expand(B, T, N).masked_fill(mask, float("-inf"))
        p = torch.softmax(logits, -1)
        return torch.cat((torch.zeros(B, T, 2, dtype=F64), p), dim=2)
    se = cfg["state_embed_dim"]
    ce = d - se
    st = (state.to(F64) @ _p(sd, pre + "state_embedder.linear.weight").T
          + _p(sd, pre + "state_embedder.linear.bias")) * math.sqrt(se)
    ca = (tgt_in_seq.to(F64) @ _p(sd, pre + "candidate_embedder.linear.weight").T
          + _p(sd, pre + "candidate_embedder.linear.bias")) * math.sqrt(ce)
    x = torch.cat((st.unsqueeze(1).expand(B, T, se), ca,
                   torch.arange(T, dtype=F64).view(1, T, 1).expand(B, T, 1)), dim=2)
    x = torch.relu(x @ _p(sd, pre + "positional_encoding_decoder.pos_embed.weight").T
                   + _p(sd, pre + "positional_encoding_decoder.pos_embed.bias"))
    causal = torch.triu(torch.ones(T, T, dtype=torch.bool), 1).expand(B, T, T)
    L, H = cfg["num_stacked_layers"], cfg["num_heads"]
    for l in range(L):
        k = f"{pre}decoder.layers.{l}."
        a, _ = _mha(x, x, _p(sd, k + "self_attn.in_proj_weight"),
                    _p(sd, k + "self_attn.in_proj_bias"), H, causal)
        a = a @ _p(sd, k + "self_attn.out_proj.weight").T + _p(sd, k + "self_attn.out_proj.bias")
        x = _ln(x + a, _p(sd, k + "norm1.weight"), _p(sd, k + "norm1.bias"))
        a, w = _mha(x, memory, _p(sd, k + "multihead_attn.in_proj_weight"),
                    _p(sd, k + "multihead_attn.in_proj_bias"), H, mask)
        if l == L - 1:
            return torch.cat((torch.zeros(B, T, 2, dtype=F64), w.mean(1)), dim=2)
        a = (a @ _p(sd, k + "multihead_attn.out_proj.weight").T
             + _p(sd, k + "multihead_attn.out_proj.bias"))
        x = _ln(x + a, _p(sd, k + "norm2.weight"), _p(sd, k + "norm2.bias"))
        f = torch.relu(x @ _p(sd, k + "linear1.weight").T + _p(sd, k + "linear1.bias"))
        f = f @ _p(sd, k + "linear2.weight").T + _p(sd, k + "linear2.bias")
        x = _ln(x + f, _p(sd, k + "norm3.weight"), _p(sd, k + "norm3.bias"))


def log_probs(sd, cfg, state, src_seq, tgt_in_idx, tgt_in_seq, tgt_out_idx):
    """(per-symbol log(clamp(p, 1e-40)) [B, T, N + 2], per-seq log(clamp(prod, 1e-40)) [B, 1])."""
    mem = encode(sd, cfg, state, src_seq)
    p = decode(sd, cfg, mem, state, tgt_in_idx, tgt_in_seq)
    seq = torch.gather(p, 2, tgt_out_idx.unsqueeze(2)).squeeze(2).prod(1, keepdim=True)
    return torch.log(p.clamp(min=1e-40)), torch.log(seq.clamp(min=1e-40))


def greedy_rank(sd, cfg, state, src_seq, T):
    """(ranked idx [B, T], per-symbol probs [B, T, N + 2], per-seq prob [B, 1]) of the greedy
    decode, re-running the decoder over the whole prefix at every step."""
    mem = encode(sd, cfg, state, src_seq)
    B, N, C = src_seq.shape
    feats = torch.cat((torch.zeros(B, 2, C, dtype=F64), src_seq.to(F64)), dim=1)
    rows = torch.arange(B).unsqueeze(1)
    if cfg["output_arch"] == "frechet_sort":
        start = torch.full((B, 1), 1, dtype=torch.long)
        p0 = decode(sd, cfg, mem, state, start, feats[rows, start])[:, 0]
        p0[:, :2] = -1.0  # never a ranked candidate
        idx = torch.sort(p0, dim=1, descending=True, stable=True).indices[:, :T]
        probs = torch.zeros(B, T, N + 2, dtype=F64).scatter(2, idx.unsqueeze(2), 1.0)
        return idx, probs, torch.ones(B, 1, dtype=F64)
    tin = torch.full((B, 1), 1, dtype=torch.long)
    probs = torch.zeros(B, T, N + 2, dtype=F64)
    for t in range(T):
        p = decode(sd, cfg, mem, state, tin, feats[rows, tin])[:, -1]
        probs[:, t] = p
        tin = torch.cat((tin, p.argmax(1, keepdim=True)), dim=1)
    idx = tin[:, 1:]
    seq = torch.gather(probs, 2, idx.unsqueeze(2)).squeeze(2).prod(1, keepdim=True)
    return idx, probs, seq.clamp(min=1e-40)


def inverse_cdf(p, u):
    """The sample rule on one step's probabilities p [B, M] and uniforms u [B]: the first j of
    nonzero probability with cumsum(p)[j] > u * sum(p), else the last j of nonzero probability
    (reached only when u * sum(p) is the total itself).  Returns (j [B], distance [B] of
    u * sum(p) to the nearest cumsum boundary between two live symbols, inf if there is none):
    a rounding smaller than that distance cannot change the choice."""
    p = p.to(F64)
    c = p.cumsum(1)
    x = u.to(F64) * c[:, -1]  # the total summed in the same order as the running sum
    live = p > 0
    M = p.shape[1]
    hit = live & (c > x.unsqueeze(1))
    last = M - 1 - live.flip(1).to(torch.int8).argmax(1)
    j = torch.where(hit.any(1), hit.to(torch.int8).argmax(1), last)
    # the boundary after the last live symbol only separates it from the fallback, which
    # picks it too
    inner = live.clone()
    inner[torch.arange(p.shape[0]), last] = False
    dist = torch.where(inner, (c - x.unsqueeze(1)).abs(), torch.full_like(c, math.inf))
    return j, dist.amin(1)


def top2_gap(probs):
    """[...]: the largest minus the second largest of probs [..., M] (the greedy choice's
    distance to a tie)."""
    top = probs.to(F64).topk(2, dim=-1).values
    return top[..., 0] - top[..., 1]


def sample_rank(sd, cfg, state, src_seq, T, noise):
    """(ranked idx [B, T], per-symbol probs [B, T, N + 2], per-seq prob [B, 1] clamped at
    1e-40, boundary distance [B, T]) of the sampled decode with uniforms noise [B, T] under the
    rule of inverse_cdf, re-running the decoder over the whole prefix at every step."""
    mem = encode(sd, cfg, state, src_seq)
    B, N, C = src_seq.shape
    feats = torch.cat((torch.zeros(B, 2, C, dtype=F64), src_seq.to(F64)), dim=1)
    rows = torch.arange(B).unsqueeze(1)
    tin = torch.full((B, 1), 1, dtype=torch.long)
    probs = torch.zeros(B, T, N + 2, dtype=F64)
    dist = torch.zeros(B, T, dtype=F64)
    for t in range(T):
        p = decode(sd, cfg, mem, state, tin, feats[rows, tin])[:, -1]
        probs[:, t] = p
        j, dist[:, t] = inverse_cdf(p, noise[:, t])
        tin = torch.cat((tin, j.unsqueeze(1)), dim=1)
    idx = tin[:, 1:]
    seq = torch.gather(probs, 2, idx.unsqueeze(2)).squeeze(2).prod(1, keepdim=True)
    return idx, probs, seq.clamp(min=1e-40), dist
