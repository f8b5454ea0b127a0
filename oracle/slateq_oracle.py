"""SlateQTrainer's update (reagent/training/slate_q_trainer.py:199-276) restated in float64 on
the CPU: next slate (SARSA or TOP_K), docs-value weighting, slate-size normalisation, discount,
target, masked MSE, torch.optim.Adam and the Polyak update.

batch (torch tensors): state [B,S], docs [B,C,D], mask / value [B,C], the same four for the
next state (next_state, next_docs, next_mask, next_value), action [B,K] and next_action
[B,K_next] int64, reward [B,K], reward_mask [B,K] bool, not_terminal [B,1] and optionally
time_diff [B,1]."""
import torch
import torch.nn.functional as F

from oracle.td_oracle import AdamState, mlp, net_params, soft_update


def to64(net, requires_grad=False):
    """A copy of an oracle net {"W", "b", "act"} in float64."""
    return {"W": [w.detach().double().clone().requires_grad_(requires_grad) for w in net["W"]],
            "b": [b.detach().double().clone().requires_grad_(requires_grad) for b in net["b"]],
            "act": list(net["act"])}


def slate_q(net, state, docs):
    """q_network(state.repeat_interleave(K), docs) viewed [B, K] for docs [B, K, D]."""
    B, K, D = docs.shape
    x = torch.cat((state.repeat_interleave(K, dim=0), docs.reshape(B * K, D)), dim=1)
    return mlp(net, x).view(B, K)


def select(t, idx):
    """DocList.select_slate of one field: t[b, idx[b, j]]."""
    return t[torch.arange(idx.shape[0]).unsqueeze(1), idx]


def docs_value(value, mask, single_selection):
    v = value * mask
    return F.softmax(v, dim=1) if single_selection else v


def head_target(q_next, next_value, next_mask, cur_mask, next_action, reward, not_terminal,
                time_diff=None, *, gamma, slate_size, maxq, single_selection, norm_next,
                time_scale=None):
    """What the loss head computes from the target network's values on EVERY next candidate,
    q_next [B,C]: (target [B,K], the next slate [B,K_next] with terminal rows zeroed).  The
    reference re-scores the chosen docs instead; the values are the same, row by row."""
    q_next, nv, nm = q_next.double(), next_value.double(), next_mask.double()
    nt = not_terminal.double().reshape(-1, 1)
    with torch.no_grad():
        if maxq:
            nxt = torch.topk(q_next * docs_value(nv, nm, single_selection), slate_size, dim=1).indices
        else:
            nxt = next_action.clone()
        nxt[nt.squeeze(1) == 0] = 0
        next_q = (select(q_next, nxt)
                  * docs_value(select(nv, nxt), select(nm, nxt), single_selection)).sum(1, keepdim=True)
        if not single_selection:
            m = nm if norm_next else cur_mask.double()
            next_q = next_q / torch.clamp(m.sum(1, keepdim=True), max=slate_size)
        discount = torch.full_like(reward.double(), gamma)
        if time_scale and time_diff is not None:
            discount = discount ** (time_diff.double().reshape(-1, 1) / time_scale)
        target = reward.double() + discount * (next_q * nt)
    return target, nxt


def head_loss(q_cur, target, reward_mask, single_selection):
    """F.mse_loss(q_cur, target), over the reward_mask entries with single selection."""
    if single_selection:
        rm = reward_mask.bool()
        return F.mse_loss(q_cur[rm], target[rm])
    return F.mse_loss(q_cur, target)


def slateq_loss(q, qt, batch, *, single_selection, **kw):
    """(loss, target, next slate) of one update; the loss carries q's autograd graph."""
    b = batch
    q_next = slate_q(qt, b["next_state"].double(), b["next_docs"].double())
    target, nxt = head_target(q_next, b["next_value"], b["next_mask"], b["mask"],
                              b["next_action"], b["reward"], b["not_terminal"], b.get("time_diff"),
                              single_selection=single_selection, **kw)
    qv = slate_q(q, b["state"].double(), select(b["docs"].double(), b["action"]))
    return head_loss(qv, target, b["reward_mask"], single_selection), target, nxt


def slateq_update(q, qt, adam: AdamState, batch, *, tau, **kw):
    """One SlateQTrainer update in place on float64 nets q (requires_grad) and qt.
    Returns (loss, grads of q, next slate)."""
    loss, _, nxt = slateq_loss(q, qt, batch, **kw)
    params = net_params(q)
    grads = [g.detach().clone() for g in torch.autograd.grad(loss, params, allow_unused=False)]
    adam.step(params, grads)
    soft_update(qt, q, tau)
    return float(loss.detach()), grads, nxt
