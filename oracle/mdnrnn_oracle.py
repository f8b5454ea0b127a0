"""Plain-torch restatement of the MDN-RNN update (reagent/models/mdn_rnn.py MDNRNN.forward and
gmm_loss, reagent/training/world_model/mdnrnn_trainer.py get_loss / configure_optimizers), with
the LSTM cell written out by hand rather than through nn.LSTM.  Runs in the dtype of its
inputs (fp64 for the host tests).

Parameters are a list in MDNRNN.parameters() order: per layer weight_ih, weight_hh, bias_ih,
bias_hh, then gmm_linear.weight and .bias.
"""
import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F

LOSS_KEYS = ("gmm", "bce", "mse", "loss")
SAMPLE_MAX = 4096  # elements per parameter kept in a golden's gradients and weights


def initial_params(seed, state_dim, action_dim, hidden, layers, gaussians):
    """The seeded initial parameters of MDNRNN(state_dim, action_dim, hidden, layers,
    gaussians) under torch.manual_seed(seed): torch's default initialisers of nn.LSTM, then of
    nn.Linear, in the order MDNRNN.__init__ builds them (fp32, parameters() order)."""
    torch.manual_seed(seed)
    rnn = torch.nn.LSTM(state_dim + action_dim, hidden, layers)
    head = torch.nn.Linear(hidden, (2 * state_dim + 1) * gaussians + 2)
    return [p.detach().clone() for p in list(rnn.parameters()) + list(head.parameters())]


def digest(t) -> np.ndarray:
    """SHA-256 of a tensor's fp32 bytes (row-major), as a uint8 array."""
    a = np.ascontiguousarray(torch.as_tensor(t).detach().cpu().float().numpy())
    return np.frombuffer(hashlib.sha256(a.tobytes()).digest(), dtype=np.uint8).copy()


def sample(t):
    """A fixed strided subsample of a tensor's elements: every ceil(n / SAMPLE_MAX)-th element
    of the flattened tensor, starting at 0 (all of them when n <= SAMPLE_MAX)."""
    flat = t.reshape(-1)
    stride = -(-flat.numel() // SAMPLE_MAX)
    return flat[::stride]


def forward(params, state, action, num_layers: int, num_gaussians: int):
    """MDNRNN.forward(action, state) from a zero initial state: the eight MemoryNetworkOutput
    fields."""
    T, B, S = state.shape
    G = num_gaussians
    H = params[1].shape[1]
    x = torch.cat([action, state], dim=-1)
    h = [x.new_zeros(B, H) for _ in range(num_layers)]
    c = [x.new_zeros(B, H) for _ in range(num_layers)]
    top = []
    for t in range(T):
        inp = x[t]
        for l in range(num_layers):
            w_ih, w_hh, b_ih, b_hh = params[4 * l: 4 * l + 4]
            gates = (h[l] @ w_hh.T + b_hh) + (inp @ w_ih.T + b_ih)
            i, f, g, o = gates.chunk(4, dim=-1)
            i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
            c[l] = f * c[l] + i * g
            h[l] = o * torch.tanh(c[l])
            inp = h[l]
        top.append(inp)
    all_h = torch.stack(top)
    y = all_h @ params[-2].T + params[-1]
    GS = G * S
    return dict(
        mus=y[:, :, :GS].reshape(T, B, G, S),
        sigmas=torch.exp(y[:, :, GS:2 * GS].reshape(T, B, G, S)),
        logpi=F.log_softmax(y[:, :, 2 * GS:2 * GS + G], dim=-1),
        reward=y[:, :, -2], not_terminal=y[:, :, -1],
        last_step_lstm_hidden=torch.stack(h), last_step_lstm_cell=torch.stack(c),
        all_steps_lstm_hidden=all_h)


def losses(out, next_state, reward, not_terminal, *, next_state_weight=1.0,
           not_terminal_weight=1.0, reward_weight=1.0, fit_only_one_next_step=False,
           state_dim=None):
    """get_loss: the mixture negative log-likelihood of next_state, the non-terminal BCE with
    logits and the reward MSE, each a mean over the rows (the last step's rows with
    fit_only_one_next_step) times its weight; loss = gmm / (state_dim + 2) + bce + mse, or
    the plain sum without state_dim."""
    mus, sigmas, logpi = out["mus"], out["sigmas"], out["logpi"]
    rs, nts = out["reward"], out["not_terminal"]
    if fit_only_one_next_step:
        next_state, not_terminal, reward = next_state[-1:], not_terminal[-1:], reward[-1:]
        mus, sigmas, logpi, rs, nts = mus[-1:], sigmas[-1:], logpi[-1:], rs[-1:], nts[-1:]
    d = next_state.unsqueeze(-2) - mus
    log_n = -(d * d) / (2 * sigmas * sigmas) - torch.log(sigmas) - math.log(math.sqrt(2 * math.pi))
    z = logpi + log_n.sum(dim=-1)
    log_prob = torch.logsumexp(z, dim=-1)
    gmm = -log_prob.mean() * next_state_weight
    bce = F.binary_cross_entropy_with_logits(nts, not_terminal) * not_terminal_weight
    mse = ((rs - reward) ** 2).mean() * reward_weight
    loss = gmm / (state_dim + 2) + bce + mse if state_dim is not None else gmm + bce + mse
    return dict(gmm=gmm, bce=bce, mse=mse, loss=loss)


def update(params, opt, batch, cfg):
    """One train_step_gen + Adam step on leaf tensors `params` with optimizer `opt`
    (torch.optim.Adam(params, lr)).  `batch`: state, action, next_state, reward,
    not_terminal.  Returns (loss dict, gradients)."""
    opt.zero_grad()
    out = forward(params, batch["state"], batch["action"], cfg["L"], cfg["G"])
    ls = losses(out, batch["next_state"], batch["reward"], batch["not_terminal"],
                next_state_weight=cfg["next_state_weight"],
                not_terminal_weight=cfg["not_terminal_weight"],
                reward_weight=cfg["reward_weight"],
                fit_only_one_next_step=cfg["fit_only_one_next_step"],
                state_dim=batch["state"].shape[2])
    ls["loss"].backward()
    grads = [p.grad.detach().clone() for p in params]
    opt.step()
    return {k: v.detach() for k, v in ls.items()}, grads
