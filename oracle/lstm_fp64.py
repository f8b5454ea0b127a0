"""Gate-level restatement of the multi-layer LSTM of the MDN-RNN and Seq2Reward networks, with
every intermediate the fused kernels keep (csrc/rb200_lstm.cuh): h and c of every layer at every
slot, the gate activations and the gate pre-activations, whose gradients are the kernels'
dGates.  Runs in the dtype of its inputs (fp64 for the tests).

The cell is the one of mdnrnn_oracle.forward and seq2reward_oracle.hidden_states, operation for
operation, so in the same dtype the outputs are theirs bit for bit:
  gates = (h . W_hh^T + b_hh) + (x . W_ih^T + b_ih),   i, f, g, o = chunk(gates, 4)
  c' = f * c + i * g,   h' = o * tanh(c')

Parameters are a list in nn.LSTM.parameters() order (per layer weight_ih, weight_hh, bias_ih,
bias_hh), optionally followed by the head's; only the first 4 * layers are read by `lstm`.
"""
import torch
import torch.nn.functional as F


def lstm(params, x, layers: int, h0=None):
    """Run the LSTM over x [T, B, K] from c0 = 0 and h0 (None: zeros; a [B, H] tensor: that h
    in every layer).  Returns a dict:
      hs, cs  [L, T+1, B, H]  slot 0 the initial state, slot t + 1 the state after step t
      acts    [L, T, B, 4H]   sigmoid(i), sigmoid(f), tanh(g), sigmoid(o)
      pre     pre[l][t] [B, 4H], the gate pre-activations; they retain their gradient, so after
              a backward `dgates(out)` is dL/dgates in the kernels' [L, T, B, 4H] layout
      top     [T, B, H] the top layer's h of every step
    hs, cs, acts and top stay connected to the graph."""
    T, B, _ = x.shape
    H = params[1].shape[1]
    if h0 is None:
        h0 = x.new_zeros(B, H)
    h = [h0 for _ in range(layers)]
    c = [torch.zeros_like(h0) for _ in range(layers)]
    hs = [[h[l]] for l in range(layers)]
    cs = [[c[l]] for l in range(layers)]
    acts = [[] for _ in range(layers)]
    pre = [[] for _ in range(layers)]
    top = []
    for t in range(T):
        inp = x[t]
        for l in range(layers):
            w_ih, w_hh, b_ih, b_hh = params[4 * l: 4 * l + 4]
            gates = (h[l] @ w_hh.T + b_hh) + (inp @ w_ih.T + b_ih)
            if gates.requires_grad:
                gates.retain_grad()
            pre[l].append(gates)
            i, f, g, o = gates.chunk(4, dim=-1)
            i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
            c[l] = f * c[l] + i * g
            h[l] = o * torch.tanh(c[l])
            acts[l].append(torch.cat([i, f, g, o], dim=-1))
            hs[l].append(h[l])
            cs[l].append(c[l])
            inp = h[l]
        top.append(inp)
    return dict(hs=torch.stack([torch.stack(v) for v in hs]),
                cs=torch.stack([torch.stack(v) for v in cs]),
                acts=torch.stack([torch.stack(v) for v in acts]), pre=pre, top=torch.stack(top))


def dgates(out):
    """[L, T, B, 4H] gradients of the gate pre-activations after a backward (zeros where the
    loss does not depend on a step)."""
    return torch.stack([torch.stack([g.grad if g.grad is not None else torch.zeros_like(g)
                                     for g in row]) for row in out["pre"]])


def input_weight_grads(out, x, layers: int):
    """The LSTM parameter gradients rebuilt from dGates, in parameters() order:
    dW_ih = sum_t dG_t^T x_t (x: the input, or h_t of the layer below), dW_hh = sum_t dG_t^T
    h_{t-1}, db_ih = db_hh = sum_t dG_t."""
    dg = dgates(out)
    hs = out["hs"].detach()
    grads = []
    for l in range(layers):
        inp = x if l == 0 else hs[l - 1, 1:]
        d = dg[l]
        grads += [torch.einsum("tbn,tbk->nk", d, inp), torch.einsum("tbn,tbk->nk", d, hs[l, :-1]),
                  d.sum((0, 1)), d.sum((0, 1))]
    return grads


def mdnrnn(params, state, action, layers: int, gaussians: int):
    """MDNRNN.forward(action, state): x = cat(action, state), the LSTM from zeros, then
    gmm_linear on the top h.  Returns `lstm`'s dict plus x, the raw head output y [T, B, NG]
    and mdnrnn_oracle.forward's fields (mus, sigmas, logpi, reward, not_terminal,
    last_step_lstm_hidden, last_step_lstm_cell, all_steps_lstm_hidden)."""
    T, B, S = state.shape
    G = gaussians
    x = torch.cat([action, state], dim=-1)
    out = lstm(params, x, layers)
    y = out["top"] @ params[4 * layers].T + params[4 * layers + 1]
    GS = G * S
    out.update(
        x=x, y=y, mus=y[:, :, :GS].reshape(T, B, G, S),
        sigmas=torch.exp(y[:, :, GS:2 * GS].reshape(T, B, G, S)),
        logpi=F.log_softmax(y[:, :, 2 * GS:2 * GS + G], dim=-1),
        reward=y[:, :, -2], not_terminal=y[:, :, -1],
        last_step_lstm_hidden=out["hs"][:, T], last_step_lstm_cell=out["cs"][:, T],
        all_steps_lstm_hidden=out["top"])
    return out


def seq2reward(params, state0, action, layers: int, valid_step=None):
    """Seq2RewardNetwork.forward: h0 = map_linear(state0) in every layer, c0 = 0, the LSTM over
    the actions, then lstm_linear on the top h of step valid_step - 1 (the last without).
    Returns `lstm`'s dict plus h0 (it retains its gradient: after a backward h0.grad is dh0,
    summed over the layers) and acc_reward [B, 1]."""
    w_lin, b_lin, w_map, b_map = params[4 * layers: 4 * layers + 4]
    h0 = state0 @ w_map.T + b_map
    if h0.requires_grad:
        h0.retain_grad()
    out = lstm(params, action, layers, h0)
    B = action.shape[1]
    top = out["top"]
    sel = top[-1] if valid_step is None else top[valid_step - 1, torch.arange(B)]
    out.update(h0=h0, acc_reward=sel @ w_lin.T + b_lin)
    return out
