"""seq2slate_kernel (csrc/rb200_seq2slate.cu) against the fp64 oracle (oracle/seq2slate_oracle.py)
at the edges of the shapes, decodes and workspaces it accepts.

* Every launch goes straight to rb200_seq2slate_forward / rb200_seq2slate_rank with outputs
  filled with NaN (indices with -7) after the workspace was allocated, and a global workspace
  filled with NaN too, so an output the kernel skips, or workspace it reads before writing it,
  cannot pass.
* Forced decode: the probabilities, log-probabilities and per-sequence log-probability against
  O.decode; columns 0 and 1 exactly 0 / log(1e-40); the log-probabilities and the sequence value
  also restated from the kernel's own probabilities.
* Rank: each step's probabilities against O.decode on the sequence the kernel ranked (teacher
  forcing reproduces the decode, so this comparison cannot diverge); every choice against the
  greedy / inverse-CDF rule on the kernel's own fp32 probabilities, bit for bit, and against the
  oracle's choice wherever its top-2 gap or CDF boundary distance exceeds MARGIN; the sequence
  value is the clamped fp32 product of the chosen probabilities; the oracle's own greedy / sampled
  trajectory wherever every one of its steps is decisive.
* The case ids name the edge: N 1, 2, 33, 63, 64 with T = N (the last step has one live symbol)
  and T = 1; one head of 128, heads of 1, 16 heads (two per warp in the last layer); L 1 and 4;
  state embeddings of 1 and d - 1; FFN 1, just below 3d and 512 > 3d; inputs of 1 and 256;
  peaked attention whose small probabilities underflow fp32; a slice of exactly 200 KiB (shared
  memory) and one 16 bytes larger (global workspace), with more slates than CTAs on each.
Measured errors are appended to $RB200_TEST_RECORD_DIR/test_measurements.jsonl when that
directory exists."""
import copy
from dataclasses import dataclass
from typing import Optional

import numpy as np
import pytest
import torch

from oracle import seq2slate_oracle as O
from reagent_b200 import _lib
from reagent_b200.core.types import PreprocessedRankingInput
from reagent_b200.models import Seq2SlateOutputArch, Seq2SlateTransformerNet
from tests.builders import _record
from tests.kernel_util import NAN
from tests.seq2slate_cases import GLOBAL_EDGE, SMEM_EDGE, SMEM_MAX, ws_slice_bytes

pytestmark = pytest.mark.gpu

AR, FS = Seq2SlateOutputArch.AUTOREGRESSIVE, Seq2SlateOutputArch.FRECHET_SORT
ARCHS = [pytest.param(AR, id="ar"), pytest.param(FS, id="frechet")]
FORCED, GREEDY, SAMPLE = (_lib.SEQ2SLATE_DECODE_FORCED, _lib.SEQ2SLATE_DECODE_GREEDY,
                          _lib.SEQ2SLATE_DECODE_SAMPLE)
LOG_FLOOR = torch.tensor(1e-40).log()    # fp32 log of the fp32 denormal 1e-40, as the kernel
LIVE = 1e-30                             # oracle probabilities whose log is compared
MARGIN = 1e-4                            # a top-2 gap or CDF distance that rounding cannot cross
ONE_BELOW = float(torch.nextafter(torch.tensor(1.0), torch.tensor(0.0)))
F64 = torch.float64


@dataclass
class Case:
    name: str
    N: int = 13
    T: int = 7
    S: int = 5
    C: int = 6
    d: int = 32
    H: int = 4
    F: int = 48
    L: int = 2
    se: Optional[int] = None
    B: int = 5
    peak: float = 0.0      # scale of the last attention scores (see _peak)
    prob: tuple = (1e-4, 1e-6)    # (rtol, atol) of probabilities
    logp: tuple = (1e-5, 2e-5)    # (rtol, atol) of log-probabilities above LIVE
    seq_rtol: float = 1e-4        # per-sequence probability against the oracle's


CASES = [
    Case("n1_t1", N=1, T=1),
    Case("n2_t2", N=2, T=2),
    Case("n2_t1", N=2, T=1),
    Case("n33_t33", N=33, T=33, B=3),
    Case("n33_t1", N=33, T=1),
    Case("n63_t63", N=63, T=63, B=2),
    Case("n63_t1", N=63, T=1),
    Case("n64_t64", N=64, T=64, B=2),
    Case("n64_t1", N=64, T=1),
    Case("h1_d128", d=128, H=1, F=96),
    Case("hd1_d8_h8", d=8, H=8),
    Case("h16_d32", d=32, H=16),
    Case("l1", L=1),
    Case("l4_h1_d128", L=4, d=128, H=1, F=160, N=21, T=9, B=3),
    Case("se1", se=1),
    Case("se31_d32", se=31),
    Case("f1", F=1),
    Case("f95_below_3d", F=95),
    Case("f512_above_3d", F=512),
    Case("s1_c1", S=1, C=1),
    Case("s256_c256", S=256, C=256),
    Case("smem_edge", S=5, B=3, **SMEM_EDGE),
    Case("global_edge", S=5, B=3, **GLOBAL_EDGE),
]
# Scores in the hundreds carry absolute fp32 errors of ~1e-5, which every probability takes on
# relatively: probabilities within atol only, and log-probabilities above LIVE within 5e-4.
# Measured on an H100 (700 W): probabilities 1.6e-5, log-probabilities 8.5e-5, sequence values
# 3.2e-5 relative.  Every other case holds the defaults: worst 1.5e-6 / 5.4e-6 relative on
# probabilities, 5.4e-6 on log-probabilities, 5.4e-6 relative on sequence values.
PEAKED = Case("peaked", N=13, T=13, B=6, peak=1.0, prob=(0.0, 1e-4), logp=(0.0, 5e-4),
              seq_rtol=5e-4)


def _net(case, arch, seed=0):
    torch.manual_seed(seed)
    net = Seq2SlateTransformerNet(state_dim=case.S, candidate_dim=case.C,
                                  num_stacked_layers=case.L, dim_model=case.d,
                                  max_src_seq_len=case.N, max_tgt_seq_len=case.T,
                                  output_arch=arch, temperature=1.0, num_heads=case.H,
                                  dim_feedforward=case.F, state_embed_dim=case.se)
    if case.peak:
        _peak(net, arch)
    return net.cuda()


@torch.no_grad()
def _peak(net, arch):
    """Sharpen the scores behind the probabilities until some live ones underflow fp32 (but
    not fp64): the last layer's query and key projections x12 (scores x144), or encoder_scorer
    x100 (score ranges of ~180)."""
    sd = net.state_dict()
    if arch == AR:
        d = net.dim_model
        sd[f"seq2slate.decoder.layers.{net.num_stacked_layers - 1}.multihead_attn."
           "in_proj_weight"][:2 * d] *= 12.0
    else:
        sd["seq2slate.encoder_scorer.weight"] *= 100.0


def _cfg(net):
    return dict(state_embed_dim=net.seq2slate.state_embed_dim, dim_model=net.dim_model,
                num_stacked_layers=net.num_stacked_layers, num_heads=net.num_heads,
                output_arch=net.output_arch.value)


def _sd(net):
    return {k: v.detach().cpu() for k, v in net.state_dict().items()}


def _inputs(case, B, seed=1):
    """state [B, S], src [B, N, C], and the teacher-forcing tensors of a random permutation
    prefix per row (CPU)."""
    g = torch.Generator().manual_seed(seed)
    state, src = torch.randn(B, case.S, generator=g), torch.randn(B, case.N, case.C, generator=g)
    action = torch.stack([torch.randperm(case.N, generator=g)[:case.T] for _ in range(B)])
    inp = PreprocessedRankingInput.from_input(state=state, candidates=src,
                                              device=torch.device("cpu"), action=action)
    return state, src, inp.tgt_in_idx, inp.tgt_out_idx, inp.tgt_in_seq.float_features


def _feats(src, tin):
    """Decoder input features of the symbols tin [B, T]: zeros for 0 / 1, else src rows."""
    B = src.shape[0]
    feats = torch.cat((torch.zeros(B, 2, src.shape[2]), src), dim=1)
    return feats[torch.arange(B).unsqueeze(1), tin]


# ------------------------------------------------------------------------------------------
# launches
# ------------------------------------------------------------------------------------------
def _poison_workspace(net):
    for ws in net._ws.values():
        ws.fill_(NAN)


def _outputs(B, T, M, n=1):
    """n sets of (ranked idx, probs, log-probs, per-sequence value), NaN / -7 filled."""
    return [(torch.full((B, T), -7, dtype=torch.int64, device="cuda"),
             torch.full((B, T, M), NAN, device="cuda"), torch.full((B, T, M), NAN, device="cuda"),
             torch.full((B,), NAN, device="cuda")) for _ in range(n)]


def _forced(net, state, src, tin, tout, tseq):
    """(probs [B, T, N + 2], log_probs, seq_log_prob [B]) of rb200_seq2slate_forward (CPU)."""
    B, N = src.shape[:2]
    T = tin.shape[1]
    st, sr = state.cuda(), src.cuda()
    a, keep = net._args(st, sr, T, FORCED)
    _poison_workspace(net)
    ins = [tin.cuda(), tout.cuda(), tseq.cuda().float().contiguous()]
    [(_, probs, logp, seq)] = _outputs(B, T, N + 2)
    a.tgt_in_idx, a.tgt_out_idx, a.tgt_in_seq = (t.data_ptr() for t in ins)
    a.probs, a.log_probs, a.seq_log_prob = probs.data_ptr(), logp.data_ptr(), seq.data_ptr()
    _lib.check(_lib.lib().rb200_seq2slate_forward(a, _lib.cur_stream()), "rb200_seq2slate_forward")
    torch.cuda.synchronize()
    del keep, ins
    return probs.cpu(), logp.cpu(), seq.cpu()


def _rank(net, state, src, T, decode, noise=None):
    """(ranked idx [B, T], probs [B, T, N + 2], seq_prob [B]) of rb200_seq2slate_rank (CPU)."""
    B, N = src.shape[:2]
    st, sr = state.cuda(), src.cuda()
    a, keep = net._args(st, sr, T, decode)
    _poison_workspace(net)
    nz = noise.cuda().float().contiguous() if noise is not None else None
    [(idx, probs, _, seq)] = _outputs(B, T, N + 2)
    if nz is not None:
        a.noise = nz.data_ptr()
    a.ranked_idx, a.probs, a.seq_prob = idx.data_ptr(), probs.data_ptr(), seq.data_ptr()
    _lib.check(_lib.lib().rb200_seq2slate_rank(a, _lib.cur_stream()), "rb200_seq2slate_rank")
    torch.cuda.synchronize()
    del keep, nz
    return idx.cpu(), probs.cpu(), seq.cpu()


def _each_row_alone(net, state, src, T, tin, tout, tseq, noise):
    """The forced and the sampled launch of every row on its own (B 1), into rows of one set
    of outputs: ((probs, log_probs, seq_log_prob), (idx, probs, seq_prob)) on the CPU."""
    B, N = src.shape[:2]
    st, sr = state.cuda(), src.cuda()
    tin, tout, tseq, nz = tin.cuda(), tout.cuda(), tseq.cuda().float().contiguous(), noise.cuda()
    (_, fp, fl, fs), (ri, rp, _, rs) = _outputs(B, T, N + 2, 2)
    lib, stream = _lib.lib(), _lib.cur_stream()
    af, keep = net._args(st[:1], sr[:1], T, FORCED)
    ar, keep2 = net._args(st[:1], sr[:1], T, SAMPLE)
    _poison_workspace(net)
    for b in range(B):
        for a in (af, ar):
            a.state, a.src_seq = st[b].data_ptr(), sr[b].data_ptr()
        af.tgt_in_idx, af.tgt_out_idx, af.tgt_in_seq = (tin[b].data_ptr(), tout[b].data_ptr(),
                                                        tseq[b].data_ptr())
        af.probs, af.log_probs = fp[b].data_ptr(), fl[b].data_ptr()
        af.seq_log_prob = fs[b:].data_ptr()
        _lib.check(lib.rb200_seq2slate_forward(af, stream), "rb200_seq2slate_forward")
        ar.noise = nz[b].data_ptr()
        ar.ranked_idx, ar.probs, ar.seq_prob = (ri[b].data_ptr(), rp[b].data_ptr(),
                                                rs[b:].data_ptr())
        _lib.check(lib.rb200_seq2slate_rank(ar, stream), "rb200_seq2slate_rank")
    torch.cuda.synchronize()
    del keep, keep2
    return (fp.cpu(), fl.cpu(), fs.cpu()), (ri.cpu(), rp.cpu(), rs.cpu())


# ------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------
class Errors:
    """Worst errors of one case: each is asserted against its bound as it is measured, and
    record() writes those measured."""

    def __init__(self, what):
        self.what, self.errs = what, {}

    def close(self, name, got, want, rtol, atol):
        g, w = got.double(), want.double()
        assert torch.isfinite(g).all(), (self.what, name, "unwritten or non-finite elements")
        err = (g - w).abs()
        self.errs[name] = dict(abs=float(err.max()) if err.numel() else 0.0,
                               rel=float((err / w.abs().clamp(min=1e-30)).max())
                               if err.numel() else 0.0)
        torch.testing.assert_close(g, w, rtol=rtol, atol=atol,
                                   msg=lambda m: f"{self.what} {name}: {m}")

    def note(self, name, value):
        self.errs[name] = value

    def record(self, test):
        _record(test, case=self.what, worst=self.errs)


def _prod32(p):
    """fp32 product of p [B, T] in step order, clamped at the fp32 denormal 1e-40 (the kernel's
    s_prod)."""
    q = np.multiply.accumulate(p.numpy().astype(np.float32), axis=1, dtype=np.float32)[:, -1]
    return torch.from_numpy(np.maximum(q, np.float32(1e-40)))


def _sample32(probs, noise):
    """The kernel's sample rule in fp32 on its own probabilities [B, T, M]: running sums in
    candidate order, u * total rounded once, the first live symbol whose running sum exceeds it,
    else the last live symbol."""
    p = probs.numpy()
    c = np.cumsum(p, axis=2, dtype=np.float32)          # sequential, as the kernel adds
    x = noise.numpy().astype(np.float32) * c[..., -1]
    live = p > 0
    hit = live & (c > x[..., None])
    last = p.shape[2] - 1 - np.argmax(live[..., ::-1], axis=2)
    return torch.from_numpy(np.where(hit.any(2), np.argmax(hit, axis=2), last))


def _check_forced(case, net, state, src, tin, tout, tseq, out, err):
    probs, logp, seq = out
    for name, t in (("probs", probs), ("log_probs", logp), ("seq_log_prob", seq)):
        assert torch.isfinite(t).all(), (err.what, name, "unwritten or non-finite elements")
    assert (probs[:, :, :2] == 0).all()
    assert (logp[:, :, :2] == LOG_FLOOR).all()
    sd, cfg = _sd(net), _cfg(net)
    ref = O.decode(sd, cfg, O.encode(sd, cfg, state, src), state, tin, tseq)
    err.close("forced.probs", probs, ref, *case.prob)
    live = ref > LIVE
    err.close("forced.log_probs", logp[live], ref[live].log(), *case.logp)
    # the log of the clamped probability everywhere (logf: within an ulp or two)
    torch.testing.assert_close(logp.double(), probs.double().clamp(min=1e-40).log(), rtol=1e-6,
                               atol=1e-6)
    chosen = torch.gather(probs, 2, tout.unsqueeze(2)).squeeze(2)
    torch.testing.assert_close(seq, _prod32(chosen).log(), rtol=1e-6, atol=0)
    oseq = torch.gather(ref, 2, tout.unsqueeze(2)).squeeze(2).prod(1).clamp(min=1e-40)
    err.close("forced.seq_prob", seq.double().exp(), oseq, case.seq_rtol, 0)
    return ref


def _check_rank(case, net, state, src, T, decode, noise, out, err):
    idx, probs, seq = out
    B, N = src.shape[:2]
    M = N + 2
    assert torch.isfinite(probs).all() and torch.isfinite(seq).all(), (err.what, "unwritten")
    assert ((idx >= 2) & (idx < M)).all(), (err.what, "ranked a padding / start symbol", idx)
    assert all(len(set(r)) == T for r in idx.tolist()), (err.what, "not a permutation prefix")
    sd, cfg = _sd(net), _cfg(net)
    mem = O.encode(sd, cfg, state, src)
    tag = "greedy" if decode == GREEDY else "sample"
    if net.output_arch == FS and decode == GREEDY:
        # the argsort of the first step's probabilities, one-hot probabilities, seq_prob 1
        assert torch.equal(probs, torch.zeros(B, T, M).scatter(2, idx.unsqueeze(2), 1.0))
        assert torch.equal(seq, torch.ones(B))
        ones = torch.ones(B, 1, dtype=torch.long)
        own = _forced(net, state, src, ones, ones + 1, torch.zeros(B, 1, src.shape[2]))[0][:, 0]
        own[:, :2] = -1.0
        assert torch.equal(idx, torch.sort(own, dim=1, descending=True, stable=True).indices[:, :T])
        p0 = O.decode(sd, cfg, mem, state, ones, _feats(src, ones))[:, 0]
        p0[:, :2] = -1.0
        so = torch.sort(p0, dim=1, descending=True, stable=True)
        gaps = so.values[:, :T] - so.values[:, 1:T + 1]
        for b in range(B):
            k = int((gaps[b] > MARGIN).to(torch.int8).argmin()) if (gaps[b] <= MARGIN).any() else T
            assert torch.equal(idx[b, :k], so.indices[b, :k]), (err.what, b, k)
        err.close("rank.step0_probs", own[:, 2:], p0[:, 2:], *case.prob)
        return
    tin = torch.cat((torch.ones(B, 1, dtype=torch.long), idx[:, :-1]), dim=1)
    ref = O.decode(sd, cfg, mem, state, tin, _feats(src, tin))
    err.close(f"{tag}.probs", probs, ref, *case.prob)
    # never a masked symbol, in either precision
    assert (torch.gather(probs, 2, idx.unsqueeze(2)) > 0).all()
    assert (torch.gather(ref, 2, idx.unsqueeze(2)) > 0).all()
    # the rule on the kernel's own fp32 probabilities, exactly
    own = torch.from_numpy(probs.numpy().argmax(2)) if decode == GREEDY else _sample32(probs, noise)
    assert torch.equal(idx, own), (err.what, "choice differs from the rule on its own probs")
    # the oracle's choice after the same prefix, wherever rounding cannot cross it
    if decode == GREEDY:
        want, margin = ref.argmax(2), O.top2_gap(ref)
    else:
        want, margin = torch.zeros(B, T, dtype=torch.long), torch.zeros(B, T, dtype=F64)
        for t in range(T):
            want[:, t], margin[:, t] = O.inverse_cdf(ref[:, t], noise[:, t])
    sure = margin > MARGIN
    assert torch.equal(idx[sure], want[sure]), (err.what, "choice differs from the oracle's")
    assert sure.double().mean() >= 0.5, (err.what, "too few decisive steps to compare")
    err.note(f"{tag}.decisive_steps", f"{int(sure.sum())}/{sure.numel()}")
    # the sequence value: the clamped fp32 product of the chosen probabilities
    chosen = torch.gather(probs, 2, idx.unsqueeze(2)).squeeze(2)
    assert torch.equal(seq, _prod32(chosen))
    oseq = torch.gather(ref, 2, idx.unsqueeze(2)).squeeze(2).prod(1).clamp(min=1e-40)
    err.close(f"{tag}.seq_prob", seq, oseq, case.seq_rtol, 0)
    # the oracle's own trajectory, on the rows where each of its steps is decisive
    if decode == GREEDY:
        oidx, oprobs, _ = O.greedy_rank(sd, cfg, state, src, T)
        osure = (O.top2_gap(oprobs) > MARGIN).all(1)
    else:
        oidx, _, _, dist = O.sample_rank(sd, cfg, state, src, T, noise)
        osure = (dist > MARGIN).all(1)
    assert torch.equal(idx[osure], oidx[osure]), (err.what, "trajectory differs from the oracle's")



# ------------------------------------------------------------------------------------------
# shapes
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("case", CASES + [PEAKED], ids=lambda c: c.name)
def test_forced_decode(case, arch):
    net = _net(case, arch)
    state, src, tin, tout, tseq = _inputs(case, case.B)
    err = Errors(f"{case.name}/{arch.value}")
    out = _forced(net, state, src, tin, tout, tseq)
    ref = _check_forced(case, net, state, src, tin, tout, tseq, out, err)
    if case.peak:
        under = (ref > 0) & (ref < 1e-45)
        assert under.any(), "the peaked case must underflow some live fp32 probabilities"
        err.note("underflowed", int(under.sum()))
    err.record("test_forced_decode")


@pytest.mark.parametrize("decode", [pytest.param(GREEDY, id="greedy"),
                                    pytest.param(SAMPLE, id="sample")])
@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("case", CASES + [PEAKED], ids=lambda c: c.name)
def test_rank(case, arch, decode):
    net = _net(case, arch)
    state, src, _, _, _ = _inputs(case, case.B)
    noise = torch.rand(case.B, case.T, generator=torch.Generator().manual_seed(9))
    err = Errors(f"{case.name}/{arch.value}")
    out = _rank(net, state, src, case.T, decode, noise if decode == SAMPLE else None)
    _check_rank(case, net, state, src, case.T, decode, noise, out, err)
    err.record("test_rank")


# ------------------------------------------------------------------------------------------
# inputs the API allows
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ARCHS)
def test_forced_repeated_input_symbols(arch):
    """tgt_in_idx may name a candidate more than once (and the start symbol anywhere): the
    cross-attention mask is the union of the inputs so far."""
    case = Case("repeats", N=9, T=9, B=6)
    net = _net(case, arch)
    state, src, _, tout, _ = _inputs(case, case.B)
    g = torch.Generator().manual_seed(3)
    tin = torch.randint(1, 6, (case.B, case.T), generator=g)  # symbols 1..5: many repeats
    tin[:, 0] = 1
    err = Errors(f"repeats/{arch.value}")
    out = _forced(net, state, src, tin, tout, _feats(src, tin))
    _check_forced(case, net, state, src, tin, tout, _feats(src, tin), out, err)
    err.record("test_forced_repeated_input_symbols")


@pytest.mark.parametrize("arch", ARCHS)
def test_forced_target_already_masked(arch):
    """A tgt_out_idx naming a symbol already fed in has probability 0 (exactly): the sequence
    log-probability is exactly log(1e-40)."""
    case = Case("masked_target", N=9, T=6, B=4)
    net = _net(case, arch)
    state, src, tin, tout, tseq = _inputs(case, case.B)
    tout = tout.clone()
    tout[:, 3] = tin[:, 2]          # fed in at step 2, masked from step 2 on
    tout[0, 5] = tin[0, 5]          # fed in at this very step
    err = Errors(f"masked_target/{arch.value}")
    out = _forced(net, state, src, tin, tout, tseq)
    _check_forced(case, net, state, src, tin, tout, tseq, out, err)
    probs, _, seq = out
    assert (probs[:, 3].gather(1, tout[:, 3:4]) == 0).all() and probs[0, 5, tout[0, 5]] == 0
    assert torch.equal(seq, LOG_FLOOR.expand(case.B))
    err.record("test_forced_target_already_masked")


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("u", [0.0, ONE_BELOW, 1.0], ids=["zero", "one_below", "one"])
def test_sample_edges_of_the_noise(arch, u):
    """noise 0 picks the first live symbol; nextafter(1, 0) the last; exactly 1 finds no running
    sum above the total and takes the fallback, the last live symbol too."""
    case = Case("noise", N=13, T=13, B=6)
    net = _net(case, arch)
    state, src, _, _, _ = _inputs(case, case.B)
    noise = torch.full((case.B, case.T), u)
    err = Errors(f"noise_{u}/{arch.value}")
    out = _rank(net, state, src, case.T, SAMPLE, noise)
    _check_rank(case, net, state, src, case.T, SAMPLE, noise, out, err)
    idx, probs, _ = out
    live = probs > 0
    first = live.to(torch.int8).argmax(2)
    last = probs.shape[2] - 1 - live.flip(2).to(torch.int8).argmax(2)
    assert torch.equal(idx, first if u == 0.0 else last)
    err.record("test_sample_edges_of_the_noise")


# ------------------------------------------------------------------------------------------
# the shared / global boundary, and more slates than CTAs
# ------------------------------------------------------------------------------------------
EDGES = {"smem": Case("smem_edge", S=5, **SMEM_EDGE),
         "global": Case("global_edge", S=5, **GLOBAL_EDGE)}


def _ctas(net, case, B):
    """(CTAs of a launch of B slates, its workspace bytes)."""
    st = torch.zeros(B, case.S, device="cuda")
    sr = torch.zeros(B, case.N, case.C, device="cuda")
    a, keep = net._args(st, sr, case.T, FORCED)
    ctas = _lib.lib().rb200_seq2slate_ctas(a)
    assert ctas > 0, _lib.lib().rb200_last_error()
    return ctas, a.workspace_bytes


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("edge", ["smem", "global"])
def test_more_slates_than_ctas(edge, arch):
    """One slate more than the grid (200 KiB slices: one CTA per SM), or two passes of
    RB200_SEQ2SLATE_MAX_CTAS and one more (global slices): every row equals a launch of that row
    alone, bit for bit, so no state carries from one slate to the next in a CTA, and the rows
    b, b + grid, b + 2 grid and the last match the oracle."""
    case = EDGES[edge]
    slice_bytes = ws_slice_bytes(**{k: getattr(case, k) for k in "N T C d H F L".split()})
    assert slice_bytes == (SMEM_MAX if edge == "smem" else SMEM_MAX + 16)
    net = _net(case, arch)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid, ws = _ctas(net, case, 4 * _lib.SEQ2SLATE_MAX_CTAS)
    if edge == "smem":
        assert ws == 0
        assert grid % sms == 0 and sms <= grid < _lib.SEQ2SLATE_MAX_CTAS  # blocks per SM x SMs
        B = grid + 1
    else:
        assert ws > 0 and grid == _lib.SEQ2SLATE_MAX_CTAS
        B = 2 * grid + 1
    assert _ctas(net, case, B)[0] == grid
    state, src, tin, tout, tseq = _inputs(case, B, seed=7)
    noise = torch.rand(B, case.T, generator=torch.Generator().manual_seed(8))
    fwd = _forced(net, state, src, tin, tout, tseq)
    rank = _rank(net, state, src, case.T, SAMPLE, noise)
    fwd1, rank1 = _each_row_alone(net, state, src, case.T, tin, tout, tseq, noise)
    for name, got, alone in zip(("probs", "log_probs", "seq_log_prob", "idx", "rank.probs",
                                 "seq_prob"), fwd + rank, fwd1 + rank1):
        same = (got == alone).reshape(B, -1).all(1)
        assert same.all(), (edge, name, "rows that differ from their own launch",
                            torch.nonzero(~same).reshape(-1)[:16].tolist())
    rows = sorted({r for r in (0, 37, 37 + grid, grid, 2 * grid, B - 1) if r < B})
    err = Errors(f"{edge}_edge_B{B}/{arch.value}")
    err.note("grid", grid)
    _check_forced(case, net, state[rows], src[rows], tin[rows], tout[rows], tseq[rows],
                  tuple(t[rows] for t in fwd), err)
    _check_rank(case, net, state[rows], src[rows], case.T, SAMPLE, noise[rows],
                tuple(t[rows] for t in rank), err)
    err.record("test_more_slates_than_ctas")


def test_workspace_cache_across_batch_sizes():
    """One net called at B 2113, then B 10, then B 2113 again on the global workspace: each
    result equals the same call on a fresh copy of the net, bit for bit."""
    case = EDGES["global"]
    net = _net(case, AR)
    B = 2 * _lib.SEQ2SLATE_MAX_CTAS + 1
    state, src, tin, tout, tseq = (t.cuda() for t in _inputs(case, B, seed=11))
    noise = torch.rand(B, case.T, device="cuda")

    def run(n, rows):
        r = n.rank(state[:rows], src[:rows], case.T, greedy=False, noise=noise[:rows])
        lp = n.log_probs(state[:rows], src[:rows], tseq[:rows], tin[:rows], tout[:rows],
                         per_symbol=True)
        return [r.ranked_tgt_out_idx, r.ranked_per_symbol_probs, r.ranked_per_seq_probs, lp]

    fresh = {rows: run(copy.deepcopy(net), rows) for rows in (B, 10)}
    for rows in (B, 10, B):
        for got, want in zip(run(net, rows), fresh[rows]):
            assert torch.equal(got, want), rows
