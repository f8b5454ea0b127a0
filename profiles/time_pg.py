"""Time one ReinforceTrainer / PPOTrainer update, fused against the same update in eager torch on
the same GPU, and the two policy-gradient kernels alone.

Workloads (one update each):
  * `reinforce_cartpole`: discrete_reinforce_cartpole_online.yaml -- S 4, A 2, [64] leaky_relu,
    gamma 0.99, normalize False, subtract_mean True -- on one trajectory of 200 steps;
  * `ppo_cartpole`: discrete_ppo_cartpole_online.yaml -- [32, 32] leaky_relu, gamma 0.99,
    Adam(1e-3, weight_decay 1e-3), ppo_batch_size 2 -- on a minibatch of two 200-step
    trajectories;
  * `ppo_large`: S 128, A 16, [256, 128] relu policy and a [256, 128] value net (reward-to-go
    baseline, normalize False), a minibatch of 16 trajectories of 512 steps.
`fused` is train_batch (REINFORCE) or _update_model (PPO); `eager` is the reference's update
written with nn.Sequential, torch.distributions.Categorical, the Python discounted_returns loop
and torch.optim.Adam, from the same weights on the same data.  Both are host-clocked over
`--updates` updates ending in a synchronise; the variants alternate over `--reps` repetitions
and the median is reported.  rb200_pg_returns and rb200_pg_head are timed alone with CUDA
events over back-to-back launches, with the arguments the trainer builds for that update (the
CartPole REINFORCE configuration subtracts the mean, PPO CartPole whitens, `ppo_large` has the
value baseline and its gradient).  The card's name, power limit and maximum SM clock are read
(queried, never set) in the same run.

    python profiles/time_pg.py --out DIR [--reps 7] [--updates 20]

Writes DIR/time_pg_<card>_<limit>w.json and prints the same JSON.  Fails without a GPU.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, card_info, cuda_device, host_steps,  # noqa: E402
                             launch_us, write_result)

SHAPES = {
    "reinforce_cartpole": dict(kind="reinforce", S=4, A=2, sizes=[64], acts=["leaky_relu"],
                               value=None, T=200, n=1, wd=0.0),
    "ppo_cartpole": dict(kind="ppo", S=4, A=2, sizes=[32, 32], acts=["leaky_relu"] * 2,
                         value=None, T=200, n=2, wd=1e-3),
    "ppo_large": dict(kind="ppo", S=128, A=16, sizes=[256, 128], acts=["relu"] * 2,
                      value=[256, 128], T=512, n=16, wd=0.0),
}
GAMMA, LR = 0.99, 1e-3


def trajectories(cfg, dev):
    import torch

    from reagent_b200.core import types as rlt

    g = torch.Generator().manual_seed(1)
    out = []
    for _ in range(cfg["n"]):
        T, S, A = cfg["T"], cfg["S"], cfg["A"]
        out.append(rlt.PolicyGradientInput(
            state=rlt.FeatureData(torch.randn(T, S, generator=g).to(dev)),
            action=torch.eye(A)[torch.randint(A, (T,), generator=g)].to(dev),
            reward=torch.randn(T, generator=g).to(dev),
            log_prob=(torch.log(torch.rand(T, generator=g) * 0.9 + 0.05)).to(dev)))
    return out


def build_fused(cfg, dev):
    import torch

    from reagent_b200.gym.policies import Policy, SoftmaxActionSampler
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import PPOTrainer, ReinforceTrainer

    torch.manual_seed(0)
    net = FullyConnectedDQN(cfg["S"], cfg["A"], cfg["sizes"], cfg["acts"]).to(dev)
    value = None
    if cfg["value"] is not None:
        value = FloatFeatureFullyConnected(cfg["S"], 1, cfg["value"],
                                           ["relu"] * len(cfg["value"])).to(dev)
    pol = Policy(scorer=net, sampler=SoftmaxActionSampler())
    opt = Optimizer__Union.default(lr=LR, weight_decay=cfg["wd"])
    if cfg["kind"] == "reinforce":
        return ReinforceTrainer(pol, gamma=GAMMA, optimizer=opt, normalize=False,
                                subtract_mean=True).to(dev)
    return PPOTrainer(pol, gamma=GAMMA, optimizer=opt, normalize=value is None, value_net=value,
                      ppo_batch_size=cfg["n"], update_freq=cfg["n"]).to(dev)


def build_eager(cfg, fused, dev):
    """The reference's update in eager torch, from the fused trainer's weights."""
    import torch

    def seq(arena_net, acts):
        layers = []
        lin = [m for m in arena_net.modules() if isinstance(m, torch.nn.Linear)]
        for i, l in enumerate(lin):
            new = torch.nn.Linear(l.in_features, l.out_features).to(dev)
            with torch.no_grad():
                new.weight.copy_(l.weight)
                new.bias.copy_(l.bias)
            layers.append(new)
            if i < len(acts):
                layers.append(torch.nn.LeakyReLU() if acts[i] == "leaky_relu" else torch.nn.ReLU())
        return torch.nn.Sequential(*layers)

    policy = seq(fused.scorer, cfg["acts"])
    value = None if cfg["value"] is None else seq(fused.value_net, ["relu"] * len(cfg["value"]))
    p_opt = torch.optim.Adam(policy.parameters(), lr=LR, weight_decay=cfg["wd"])
    v_opt = None if value is None else torch.optim.Adam(value.parameters(), lr=LR)

    def discounted_returns(r):
        returns = torch.empty_like(r)
        running = torch.zeros((), device=r.device)
        for t in range(r.shape[0] - 1, -1, -1):
            running = r[t] + GAMMA * running
            returns[t] = running
        return returns

    def update(trajs):
        ppo, vl = [], []
        for t in trajs:
            s = t.state.float_features
            scores = policy(s)
            d = torch.distributions.Categorical(logits=scores / 1.0)
            lp = d.log_prob(t.action.argmax(dim=1))
            adv = discounted_returns(torch.clamp(t.reward, max=1e6))
            if cfg["kind"] == "reinforce":
                adv = adv - adv.mean()
                ppo.append(-(adv.detach() @ lp))
                continue
            if value is None:
                adv = (adv - adv.mean()) / (adv.std(unbiased=False) + 2.220446049250313e-16)
            else:
                base = value(s).reshape(-1)
                vl.append(torch.nn.functional.mse_loss(base, adv, reduction="sum"))
                adv = adv - base.detach()
            rho = torch.exp(lp - t.log_prob)
            ppo.append(-torch.min(adv * rho, adv * torch.clamp(rho, 0.8, 1.2)).sum())
        if value is not None:
            v_opt.zero_grad()
            torch.stack(vl).sum().backward()
            v_opt.step()
        loss = torch.stack(ppo).sum()
        p_opt.zero_grad()
        loss.backward()
        p_opt.step()
        return loss.detach()

    return update


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--updates", type=int, default=20)
    args = ap.parse_args(argv)
    dev = cuda_device(__file__)
    import torch

    from reagent_b200 import _lib

    torch.distributions.Distribution.set_default_validate_args(False)
    res = {"card": card_info(), "method": (
        "host-clocked updates ending in a synchronise, fused and eager alternating; kernels "
        "alone: CUDA events over back-to-back launches"), "update_us": {}, "kernel_us": {}}
    for name, cfg in SHAPES.items():
        fused = build_fused(cfg, dev)
        trajs = trajectories(cfg, dev)
        eager = build_eager(cfg, fused, dev)
        if cfg["kind"] == "reinforce":
            fused_step = lambda i: fused.train_batch(trajs[0], i)  # noqa: E731
        else:
            def fused_step(i):
                fused._update_model(trajs)
                return fused.last_losses
        steps = {"fused": fused_step, "eager": lambda i: eager(trajs)}
        for f in steps.values():
            host_steps(f, 3)  # warm-up: module loads, allocations
        res["update_us"][name] = alternate(
            ["fused", "eager"], args.reps, lambda k, rep: host_steps(steps[k], args.updates)[0])
        # the two kernels alone, with the arguments the trainer builds for this update
        batch = trajs[0] if cfg["kind"] == "reinforce" else trajs
        p, pins = fused._pack(batch)
        kw = fused._settings(p)
        fused._pg.run(p, pins, **kw)  # fills the scores and values the head reads
        ws = fused._pg.ws
        r = fused._pg.returns_args(p, ws, **kw)
        h = fused._pg.head_args(p, ws, **kw)
        st = _lib.cur_stream()
        lib = _lib.lib()
        res["kernel_us"][name] = alternate(["returns", "head"], args.reps, lambda k, rep: launch_us(
            (lambda: lib.rb200_pg_returns(r, st)) if k == "returns"
            else (lambda: lib.rb200_pg_head(h, st)), 200))
        del pins
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
