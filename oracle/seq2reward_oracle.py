"""Plain-torch restatement of Seq2Reward (reagent/models/seq2reward_model.py forward,
reagent/training/world_model/seq2reward_trainer.py get_mse_loss / get_step_entropy_loss /
get_Q, compress_model_trainer.py get_loss), with the LSTM cell written out by hand rather than
through nn.LSTM.  Runs in the dtype of its inputs (fp64 for the tests); gradients come from
autograd through these formulas.

Parameters are a list in Seq2RewardNetwork.parameters() order: per layer weight_ih, weight_hh,
bias_ih, bias_hh, then lstm_linear.weight and .bias, then map_linear.weight and .bias.
"""
import itertools

import torch
import torch.nn.functional as F


def initial_params(seed, state_dim, action_dim, hidden, layers):
    """The seeded initial parameters of Seq2RewardNetwork under torch.manual_seed(seed): torch's
    default initialisers of nn.LSTM, lstm_linear and map_linear, in that order (fp32)."""
    torch.manual_seed(seed)
    rnn = torch.nn.LSTM(action_dim, hidden, layers)
    lstm_linear = torch.nn.Linear(hidden, 1)
    map_linear = torch.nn.Linear(state_dim, hidden)
    mods = list(rnn.parameters()) + list(lstm_linear.parameters()) + list(map_linear.parameters())
    return [p.detach().clone() for p in mods]


def hidden_states(params, state0, action, layers: int):
    """Top-layer h of every step [T, B, H]: h0 = map_linear(state0) in every layer, c0 = 0."""
    w_lin, b_lin, w_map, b_map = params[4 * layers:]
    h0 = state0 @ w_map.T + b_map
    h = [h0 for _ in range(layers)]
    c = [torch.zeros_like(h0) for _ in range(layers)]
    tops = []
    for t in range(action.shape[0]):
        x = action[t]
        for l in range(layers):
            w_ih, w_hh, b_ih, b_hh = params[4 * l: 4 * l + 4]
            gates = (h[l] @ w_hh.T + b_hh) + (x @ w_ih.T + b_ih)
            i, f, g, o = gates.chunk(4, dim=1)
            i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
            c[l] = f * c[l] + i * g
            h[l] = o * torch.tanh(c[l])
            x = h[l]
        tops.append(x)
    return torch.stack(tops)


def forward(params, state0, action, layers: int, valid_step=None):
    """acc_reward [B, 1]: lstm_linear on the top h of step valid_step - 1 (the last without)."""
    w_lin, b_lin = params[4 * layers: 4 * layers + 2]
    tops = hidden_states(params, state0, action, layers)
    B = action.shape[1]
    sel = tops[-1] if valid_step is None else tops[valid_step - 1, torch.arange(B)]
    return sel @ w_lin.T + b_lin


def target(reward, valid_step, gamma: float):
    """cumsum(reward * fp32(gamma ** t))[valid - 1], summed in fp64 (torch's CPU cumsum)."""
    T, B = reward.shape
    mask = torch.tensor([gamma ** i for i in range(T)], dtype=torch.float32).to(reward.dtype)
    prod = reward.float() * mask.float()[:, None]
    acc = torch.cumsum(prod.double(), dim=0)
    return acc[valid_step - 1, torch.arange(B)].unsqueeze(1)


def mse_loss(params, state0, action, reward, valid_step, layers: int, gamma: float):
    pred = forward(params, state0, action, layers, valid_step)
    return F.mse_loss(pred, target(reward, valid_step, gamma).to(pred.dtype))


def mlp(params, x, acts):
    """An MLP given [W0, b0, W1, b1, ...] and activation names."""
    for l, a in enumerate(acts):
        x = x @ params[2 * l].T + params[2 * l + 1]
        x = torch.relu(x) if a == "relu" else x
    return x


def step_loss(step_params, state0, valid_step):
    """get_step_entropy_loss: cross entropy of the step MLP against valid_step - 1."""
    logits = mlp(step_params, state0, ["relu", "relu", "linear"])
    return F.cross_entropy(logits, valid_step - 1)


def grads(loss, params):
    return torch.autograd.grad(loss, params)


def permutations(seq_len: int, num_action: int):
    """Every action sequence of length seq_len in lexical order, as index tuples."""
    return list(itertools.product(range(num_action), repeat=seq_len))


def get_q(params, state, num_action: int, seq_len: int, layers: int):
    """[B, A]: max over the sequences starting with each action of the predicted reward, by
    flat enumeration (one forward over every (state, sequence) pair)."""
    B = state.shape[0]
    seqs = torch.tensor(permutations(seq_len, num_action)).T  # [k, n]
    n = seqs.shape[1]
    act = F.one_hot(seqs, num_action).to(state.dtype).repeat(1, B, 1)  # [k, B * n, A]
    s = state.repeat_interleave(n, dim=0)
    r = forward(params, s, act, layers).reshape(B, num_action, n // num_action)
    return r.max(dim=2).values


def get_q_all(params, state, num_action: int, seq_len: int, layers: int):
    """[B, k, A]: get_q at every horizon 1..k."""
    return torch.stack([get_q(params, state, num_action, j, layers)
                        for j in range(1, seq_len + 1)], dim=1)


def compress(out, q):
    """(mse, accuracy) of CompressModelTrainer.get_loss; argmax keeps the first maximum."""
    mse = F.mse_loss(out, q)
    acc = torch.mean((first_argmax(q) == first_argmax(out)).to(out.dtype))
    return mse, acc


def first_argmax(x):
    """Index of the first maximum of each row."""
    m = x.max(dim=1, keepdim=True).values
    idx = torch.arange(x.shape[1]).expand_as(x)
    return torch.where(x == m, idx, x.shape[1]).min(dim=1).values
