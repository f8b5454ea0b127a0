"""torch.optim.AdamW with optional AMSGrad, restated next to td_oracle.AdamState (which is
torch.optim.Adam).  The reference's CartPole QR-DQN and C51 configurations select it with
`AdamW: {lr: 0.001, amsgrad: true}` (reagent/optimizer/uninferrable_optimizers.py:70-78).
Follows torch's single-tensor path (torch/optim/adam.py, _single_tensor_adam, with
decoupled_weight_decay=True): the parameters decay before the moment updates, and with AMSGrad
the denominator uses the running maximum of exp_avg_sq."""
import torch

from oracle.td_oracle import AdamState


class AdamWState(AdamState):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                 amsgrad=False):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        self.amsgrad = amsgrad
        self.vmax = [torch.zeros_like(p) for p in params] if amsgrad else None

    @torch.no_grad()
    def step(self, params, grads):
        self.t += 1
        b1, b2 = self.betas
        bc1 = 1 - b1 ** self.t
        bc2 = 1 - b2 ** self.t
        step_size = self.lr / bc1
        bc2_sqrt = bc2 ** 0.5
        for i, (p, g, m, v) in enumerate(zip(params, grads, self.m, self.v)):
            if self.wd != 0:
                p.mul_(1 - self.lr * self.wd)
            m.lerp_(g, 1 - b1)
            v.mul_(b2).addcmul_(g, g, value=1 - b2)
            d = v
            if self.amsgrad:
                torch.maximum(self.vmax[i], v, out=self.vmax[i])
                d = self.vmax[i]
            denom = (d.sqrt() / bc2_sqrt).add_(self.eps)
            p.addcdiv_(m, denom, value=-step_size)
