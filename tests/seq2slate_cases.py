"""The Seq2Slate golden cases (oracle/make_seq2slate_golden.py) as torch tensors."""
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["seq2slate_autoregressive", "seq2slate_frechet_sort", "seq2slate_tsp", "seq2slate_odd"]


def load(name):
    """(meta, {array name: tensor}, state_dict)"""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(bytes(z["__meta__"]).decode())
    arrays = {k: torch.from_numpy(z[k]) for k in z.files if k != "__meta__"}
    sd = {k[2:]: v for k, v in arrays.items() if k.startswith("p.")}
    return meta, arrays, sd


SMEM_MAX = 200 * 1024  # kS2sSmemMax: the largest per-CTA slice kept in shared memory

# Shapes at the shared / global workspace boundary (re-derive them from ws_slice_bytes if the
# slice layout changes): a slice of exactly SMEM_MAX bytes, and one 16-byte group above it.
SMEM_EDGE = dict(N=56, T=56, C=8, d=64, H=8, F=256, L=2)
GLOBAL_EDGE = dict(N=39, T=39, C=64, d=128, H=4, F=512, L=1)


def ws_slice_bytes(N, T, C, d, H, F, L):
    """Bytes of one CTA's workspace slice (s2s_ws_floats in csrc/rb200_seq2slate.cu): the
    activations X, Z [N, d] and Y [N, max(3d, F)], the cross-attention keys / values [L, N, 2d],
    the self-attention cache [L, T, 2d], the last layer's head weights [H, N], the scores [N],
    four d-rows, one max(3d, F)-row and one feature row [C], each rounded up to 4 floats."""
    r4 = lambda n: (n + 3) & ~3
    wide = max(3 * d, F)
    return 4 * (2 * r4(N * d) + r4(N * wide) + r4(L * 2 * N * d) + r4(L * 2 * T * d)
                + r4(H * N) + r4(N) + 4 * r4(d) + r4(wide) + r4(C))


def workspace_bytes(B, max_ctas, **shape):
    """rb200_seq2slate_workspace_bytes: 0 on the shared-memory path, else one slice per CTA
    for min(B, max_ctas) CTAs."""
    s = ws_slice_bytes(**shape)
    return 0 if s <= SMEM_MAX else min(B, max_ctas) * s


def build_net(meta, sd, device="cuda"):
    from reagent_b200.models import Seq2SlateOutputArch, Seq2SlateTransformerNet

    kw = {k: meta[k] for k in ("state_dim", "candidate_dim", "num_stacked_layers", "dim_model",
                               "max_src_seq_len", "max_tgt_seq_len", "temperature", "num_heads",
                               "dim_feedforward")}
    net = Seq2SlateTransformerNet(output_arch=Seq2SlateOutputArch(meta["output_arch"]),
                                  state_embed_dim=meta.get("state_embed_dim"), **kw).to(device)
    net.load_state_dict(sd)
    return net
