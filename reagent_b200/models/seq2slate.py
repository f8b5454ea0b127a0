"""Seq2SlateTransformerNet (reagent/models/seq2slate.py): a transformer encoder over the
candidates (each concatenated with the state's embedding) and a pointer decoder that emits a
permutation of them one symbol at a time.

The sub-modules are the reference's, built in its order -- torch's TransformerEncoder and
TransformerDecoderLayers, encoder_scorer, the positional encoding and the two embedders -- then
xavier-initialised in parameters() order, so `state_dict()` keys and the seeded initial weights
are its own.  The parameters are views of one flat arena.  Every mode is ONE launch of
csrc/rb200_seq2slate.cu: the log-probability modes run the teacher-forced decoder, RANK_MODE the
whole T-step decode with cached keys and values; torch's transformer layers never run.
"""
import copy
from enum import Enum
from typing import Optional

import torch
import torch.nn as nn

from .. import _lib
from ..core import types as rlt
from .arena import ParamArena, _align4
from .base import ModelBase

PADDING_SYMBOL = rlt.PADDING_SYMBOL
DECODER_START_SYMBOL = rlt.DECODER_START_SYMBOL


class Seq2SlateMode(Enum):
    RANK_MODE = "rank"
    PER_SEQ_LOG_PROB_MODE = "per_sequence_log_prob"
    PER_SYMBOL_LOG_PROB_DIST_MODE = "per_symbol_log_prob_dist"
    DECODE_ONE_STEP_MODE = "decode_one_step"
    ENCODER_SCORE_MODE = "encoder_score_mode"


class Seq2SlateOutputArch(Enum):
    # only output encoder scores (not supported here)
    ENCODER_SCORE = "encoder_score"
    # a decoder outputs a sequence in an autoregressive way
    AUTOREGRESSIVE = "autoregressive"
    # iterative softmax over the encoder scores (frechet sort)
    FRECHET_SORT = "frechet_sort"


_ARCH = {Seq2SlateOutputArch.AUTOREGRESSIVE: _lib.SEQ2SLATE_ARCH_AUTOREGRESSIVE,
         Seq2SlateOutputArch.FRECHET_SORT: _lib.SEQ2SLATE_ARCH_FRECHET_SORT}


def check_shape(state_dim, candidate_dim, state_embed_dim, dim_model, num_heads,
                dim_feedforward, num_stacked_layers, max_src_seq_len, max_tgt_seq_len):
    """Raise ValueError if the fused kernels do not take this shape (limits:
    include/reagent_b200.h)."""
    rc = _lib.lib().rb200_seq2slate_check_shape(state_dim, candidate_dim, state_embed_dim,
                                                dim_model, num_heads, dim_feedforward,
                                                num_stacked_layers, max_src_seq_len,
                                                max_tgt_seq_len)
    if rc != 0:
        raise ValueError("Seq2SlateTransformerNet: "
                         + _lib.lib().rb200_last_error().decode("utf-8", "replace"))


class ShapeArena(ParamArena):
    """Flat layout of an arbitrary parameter list, each tensor on a 16-byte boundary."""

    def __init__(self, shapes):
        self.dims, self.acts, self.w_off, self.b_off = [], [], [], []
        self.shapes = [tuple(s) for s in shapes]
        self.offsets, off = [], 0
        for s in self.shapes:
            self.offsets.append(off)
            off = _align4(off + int(torch.Size(s).numel()))
        self.n = off
        self.flat = None
        self.gpart = None
        self.grad_ready = False
        self._desc = None

    def flatten(self, params, device=None):
        """Copy `params` into a fresh flat buffer and re-point their `.data` at views of it."""
        params = list(params)
        assert [tuple(p.shape) for p in params] == self.shapes
        dev = device if device is not None else params[0].device
        flat = torch.zeros(self.n, dtype=torch.float32, device=dev)
        for p, off, s in zip(params, self.offsets, self.shapes):
            v = flat[off: off + p.numel()].view(s)
            v.copy_(p.data.to(dev, torch.float32))
            p.data = v
            p._rb200_arena = self
        self.flat = flat
        self.gpart = None
        self.grad_ready = False
        return flat


class _Embedder(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.dim_in, self.dim_out = dim_in, dim_out
        self.linear = nn.Linear(dim_in, dim_out)


class _PositionalEncoding(nn.Module):
    def __init__(self, dim_model):
        super().__init__()
        self.pos_embed = nn.Linear(dim_model + 1, dim_model)


class _EncoderPyTorch(nn.Module):
    def __init__(self, dim_model, num_heads, dim_feedforward, num_layers):
        super().__init__()
        layer = nn.TransformerEncoderLayer(d_model=dim_model, dim_feedforward=dim_feedforward,
                                           nhead=num_heads, dropout=0.0)
        self.transformer_encoder = nn.TransformerEncoder(layer, num_layers=num_layers,
                                                         enable_nested_tensor=False)


class _DecoderPyTorch(nn.Module):
    def __init__(self, dim_model, num_heads, dim_feedforward, num_layers):
        super().__init__()
        # the last layer is the reference's DecoderLastLayerPytorch: the same parameters
        self.layers = nn.ModuleList([
            nn.TransformerDecoderLayer(d_model=dim_model, nhead=num_heads,
                                       dim_feedforward=dim_feedforward, dropout=0.0)
            for _ in range(num_layers)])
        self.num_layers = num_layers


class Seq2SlateTransformerModel(nn.Module):
    """The parameter container of the reference's Seq2SlateTransformerModel."""

    def __init__(self, state_dim, candidate_dim, num_stacked_layers, num_heads, dim_model,
                 dim_feedforward, max_src_seq_len, max_tgt_seq_len, output_arch,
                 temperature=1.0, state_embed_dim=None):
        super().__init__()
        self.state_dim, self.candidate_dim = state_dim, candidate_dim
        self.num_stacked_layers, self.num_heads = num_stacked_layers, num_heads
        self.dim_model, self.dim_feedforward = dim_model, dim_feedforward
        self.max_src_seq_len, self.max_tgt_seq_len = max_src_seq_len, max_tgt_seq_len
        self.output_arch = output_arch
        self.temperature = temperature  # stored, never applied (as in the reference)
        self.encoder = _EncoderPyTorch(dim_model, num_heads, dim_feedforward, num_stacked_layers)
        self.encoder_scorer = nn.Linear(dim_model, 1)
        self.decoder = _DecoderPyTorch(dim_model, num_heads, dim_feedforward, num_stacked_layers)
        self.positional_encoding_decoder = _PositionalEncoding(dim_model)
        if state_embed_dim is None:
            state_embed_dim = dim_model // 2
        self.state_embed_dim = state_embed_dim
        self.state_embedder = _Embedder(state_dim, state_embed_dim)
        self.candidate_embedder = _Embedder(candidate_dim, dim_model - state_embed_dim)
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)


class Seq2SlateTransformerNet(ModelBase):
    def __init__(self, state_dim: int, candidate_dim: int, num_stacked_layers: int,
                 dim_model: int, max_src_seq_len: int, max_tgt_seq_len: int,
                 output_arch: Seq2SlateOutputArch, temperature: float, num_heads: int,
                 dim_feedforward: int, state_embed_dim: Optional[int] = None) -> None:
        super().__init__()
        if output_arch not in _ARCH:
            raise NotImplementedError(f"Seq2SlateTransformerNet: output_arch {output_arch} is not "
                                      "supported (AUTOREGRESSIVE and FRECHET_SORT are)")
        se = dim_model // 2 if state_embed_dim is None else state_embed_dim
        check_shape(state_dim, candidate_dim, se, dim_model, num_heads, dim_feedforward,
                    num_stacked_layers, max_src_seq_len, max_tgt_seq_len)
        self.state_dim, self.candidate_dim = state_dim, candidate_dim
        self.num_stacked_layers, self.dim_model = num_stacked_layers, dim_model
        self.max_src_seq_len, self.max_tgt_seq_len = max_src_seq_len, max_tgt_seq_len
        self.output_arch, self.temperature = output_arch, temperature
        self.num_heads, self.dim_feedforward = num_heads, dim_feedforward
        self.state_embed_dim = state_embed_dim
        self.seq2slate = Seq2SlateTransformerModel(
            state_dim=state_dim, candidate_dim=candidate_dim,
            num_stacked_layers=num_stacked_layers, num_heads=num_heads, dim_model=dim_model,
            dim_feedforward=dim_feedforward, max_src_seq_len=max_src_seq_len,
            max_tgt_seq_len=max_tgt_seq_len, output_arch=output_arch, temperature=temperature,
            state_embed_dim=state_embed_dim)
        self._arena = ShapeArena([p.shape for p in self.parameters()])
        self._arena.flatten(self.parameters())
        self._ws = {}

    @property
    def arena(self) -> ShapeArena:
        return self._arena

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        self._arena.flatten(self.parameters())
        self._ws = {}
        return self

    def __deepcopy__(self, memo):
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k not in ("_arena", "_ws"):
                new.__dict__[k] = copy.deepcopy(v, memo)
        new._arena = ShapeArena(self._arena.shapes)
        new._arena.flatten(new.parameters())
        new._ws = {}
        return new

    def input_prototype(self):
        return rlt.PreprocessedRankingInput.from_tensors(
            state=torch.randn(1, self.state_dim),
            src_seq=torch.randn(1, self.max_src_seq_len, self.candidate_dim),
            tgt_in_seq=torch.randn(1, self.max_tgt_seq_len, self.candidate_dim),
            tgt_out_seq=torch.randn(1, self.max_tgt_seq_len, self.candidate_dim),
            slate_reward=torch.randn(1))

    # -- kernel arguments ------------------------------------------------------
    def _args(self, state, src_seq, T, decode):
        B, N = src_seq.shape[0], src_seq.shape[1]
        m = self.seq2slate
        check_shape(self.state_dim, self.candidate_dim, m.state_embed_dim, self.dim_model,
                    self.num_heads, self.dim_feedforward, self.num_stacked_layers, N, T)
        state = _cuda(state, "state", (B, self.state_dim))
        src_seq = _cuda(src_seq, "src_seq", (B, N, self.candidate_dim))
        _lib.require_current_device(state.device)
        a = _lib.Seq2slateArgsT()
        a.batch, a.src_len, a.tgt_len = B, N, T
        a.state_dim, a.candidate_dim, a.state_embed_dim = (self.state_dim, self.candidate_dim,
                                                           m.state_embed_dim)
        a.dim_model, a.num_heads, a.dim_feedforward = self.dim_model, self.num_heads, self.dim_feedforward
        a.layers, a.arch, a.decode = self.num_stacked_layers, _ARCH[self.output_arch], decode
        ar = self._arena
        a.params, a.n_params = ar.flat.data_ptr(), ar.n
        for i, o in enumerate(ar.offsets):
            a.off[i] = o
        a.state, a.src_seq = state.data_ptr(), src_seq.data_ptr()
        nbytes = int(_lib.lib().rb200_seq2slate_workspace_bytes(a))
        key = (state.device, nbytes)
        ws = self._ws.get(key)
        if ws is None:
            self._ws.clear()
            ws = self._ws[key] = torch.empty(max(nbytes // 4, 1), device=state.device)
        # a launch on another stream than the allocating one keeps the buffer from being reused
        # by the caching allocator until that stream's work is done, when the cache drops it
        ws.record_stream(torch.cuda.current_stream(state.device))
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        return a, [state, src_seq]

    # -- modes -----------------------------------------------------------------
    def forward(self, input: rlt.PreprocessedRankingInput, mode: Seq2SlateMode,
                tgt_seq_len: Optional[int] = None, greedy: Optional[bool] = None,
                noise: Optional[torch.Tensor] = None) -> rlt.RankingOutput:
        if mode == Seq2SlateMode.RANK_MODE:
            assert greedy is not None
            return self.rank(input.state.float_features, input.src_seq.float_features,
                             tgt_seq_len, greedy, noise)
        if mode in (Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE,
                    Seq2SlateMode.PER_SEQ_LOG_PROB_MODE):
            assert input.tgt_in_seq is not None
            assert input.tgt_in_idx is not None
            assert input.tgt_out_idx is not None
            per_symbol = mode == Seq2SlateMode.PER_SYMBOL_LOG_PROB_DIST_MODE
            out = self.log_probs(input.state.float_features, input.src_seq.float_features,
                                 input.tgt_in_seq.float_features, input.tgt_in_idx,
                                 input.tgt_out_idx, per_symbol=per_symbol)
            return rlt.RankingOutput(log_probs=out)
        raise NotImplementedError(f"Seq2SlateTransformerNet: mode {mode} is not supported")

    def log_probs(self, state, src_seq, tgt_in_seq, tgt_in_idx, tgt_out_idx,
                  per_symbol: bool = False) -> torch.Tensor:
        """Teacher-forced decode: per-symbol log(clamp(probs, 1e-40)) [B, T, N + 2], or the
        per-sequence log(clamp(prod of the tgt_out_idx probabilities, 1e-40)) [B, 1]."""
        B, N = src_seq.shape[0], src_seq.shape[1]
        T = tgt_in_idx.shape[1]
        if T > N:
            raise ValueError(f"Seq2SlateTransformerNet: tgt_seq_len {T} > src_seq_len {N}")
        a, keep = self._args(state, src_seq, T, _lib.SEQ2SLATE_DECODE_FORCED)
        dev = keep[0].device
        tin = _index(tgt_in_idx, "tgt_in_idx", (B, T), dev)
        tout = _index(tgt_out_idx, "tgt_out_idx", (B, T), dev)
        tseq = _cuda(tgt_in_seq, "tgt_in_seq", (B, T, self.candidate_dim))
        keep += [tin, tout, tseq]
        a.tgt_in_idx, a.tgt_out_idx, a.tgt_in_seq = tin.data_ptr(), tout.data_ptr(), tseq.data_ptr()
        if per_symbol:
            out = torch.empty(B, T, N + 2, device=dev)
            a.log_probs = out.data_ptr()
        else:
            out = torch.empty(B, 1, device=dev)
            a.seq_log_prob = out.data_ptr()
        _lib.check(_lib.lib().rb200_seq2slate_forward(a, _lib.cur_stream()),
                   "rb200_seq2slate_forward")
        return out

    @torch.no_grad()
    def rank(self, state, src_seq, tgt_seq_len: Optional[int] = None, greedy: bool = True,
             noise: Optional[torch.Tensor] = None) -> rlt.RankingOutput:
        """Decode tgt_seq_len symbols (default max_tgt_seq_len) in one launch.  Sampling draws
        one uniform per (row, step) from torch's generator on the device, or reads the given
        `noise` [B, tgt_seq_len]; no host synchronisation either way."""
        B, N = src_seq.shape[0], src_seq.shape[1]
        T = self.max_tgt_seq_len if tgt_seq_len is None else int(tgt_seq_len)
        decode = _lib.SEQ2SLATE_DECODE_GREEDY if greedy else _lib.SEQ2SLATE_DECODE_SAMPLE
        a, keep = self._args(state, src_seq, T, decode)
        dev = keep[0].device
        if not greedy:
            if noise is None:
                noise = torch.rand(B, T, device=dev)
            noise = _cuda(noise, "noise", (B, T))
            keep.append(noise)
            a.noise = noise.data_ptr()
        idx = torch.empty(B, T, dtype=torch.int64, device=dev)
        probs = torch.empty(B, T, N + 2, device=dev)
        seq = torch.empty(B, 1, device=dev)
        a.ranked_idx, a.probs, a.seq_prob = idx.data_ptr(), probs.data_ptr(), seq.data_ptr()
        _lib.check(_lib.lib().rb200_seq2slate_rank(a, _lib.cur_stream()), "rb200_seq2slate_rank")
        return rlt.RankingOutput(ranked_tgt_out_idx=idx, ranked_per_symbol_probs=probs,
                                 ranked_per_seq_probs=seq)


def _cuda(t: torch.Tensor, name: str, shape) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.Rb200Error(f"Seq2SlateTransformerNet: {name} is a {t.device} tensor; "
                              "reagent_b200 runs on CUDA only (there is no CPU path)")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"Seq2SlateTransformerNet: {name} has shape {tuple(t.shape)}, "
                         f"expected {tuple(shape)}")
    return t.float().contiguous()


def _index(t: torch.Tensor, name: str, shape, device) -> torch.Tensor:
    if tuple(t.shape) != tuple(shape) or t.device != device:
        raise ValueError(f"Seq2SlateTransformerNet: {name} must be {tuple(shape)} on {device}, "
                         f"got {tuple(t.shape)} on {t.device}")
    return t.to(torch.int64).contiguous()
