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


def build_net(meta, sd, device="cuda"):
    from reagent_b200.models import Seq2SlateOutputArch, Seq2SlateTransformerNet

    kw = {k: meta[k] for k in ("state_dim", "candidate_dim", "num_stacked_layers", "dim_model",
                               "max_src_seq_len", "max_tgt_seq_len", "temperature", "num_heads",
                               "dim_feedforward")}
    net = Seq2SlateTransformerNet(output_arch=Seq2SlateOutputArch(meta["output_arch"]),
                                  state_embed_dim=meta.get("state_embed_dim"), **kw).to(device)
    net.load_state_dict(sd)
    return net
