"""Time DiscreteCRRTrainer.train_batch against the same update written in eager torch, the two
CRR loss heads alone, and the captured online FusedDqnStep step.

Shapes: the reference's CartPole configuration (S 4, A 2, B 256, [1024, 1024] relu actor and twin
FullyConnected critics, exploration_variance 1e-7) and config-2 shapes (S 128, A 16, B 4096,
[256, 128], twin critics, no exploration noise).  Per shape, in one process:
  * `fused`: DiscreteCRRTrainer.train_batch;
  * `eager`: nn.Sequential networks, torch.distributions.Categorical, F.mse_loss, autograd and
    torch.optim.Adam(capturable=True), with the soft updates as torch._foreach ops and the
    distributions' host-synchronising argument checks off (they cannot be captured), from the same
    initial weights on the same data.
Each is captured into a CUDA graph of `--calls` consecutive updates after warm-up; a run is one
replay between two CUDA events, the variants alternate, and the median of `--reps` runs is
reported per update.  The heads are timed the same way on the fused trainer's workspace.  The
online step is FusedDqnStep(rng="device", online=True).step(transition), host-timed over
`--steps` steps that end in a synchronise.  The card's name, power limit and maximum SM clock are
read (queried, never set) in the same run and name the output file.

    python profiles/time_crr.py --out DIR [--reps 7] [--calls 50]

Writes DIR/time_crr_<card>_<limit>w.json and prints the same JSON.  Fails without a GPU.
"""
import argparse
import json
import os
import re
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.time_bcq import card_info  # noqa: E402

SHAPES = {
    "cartpole": dict(S=4, A=2, B=256, sizes=[1024, 1024], noise=1e-7, gamma=0.99, tau=0.2),
    "config2": dict(S=128, A=16, B=4096, sizes=[256, 128], noise=None, gamma=0.99, tau=0.005),
}
LR = 1e-3


def algorithmic_bytes(cfg):
    """Bytes each head has to move per launch, from the shapes."""
    B, A = cfg["B"], cfg["A"]
    noise = 0 if cfg["noise"] is None else 1
    critic = 4 * (B * A * (6 + noise) + 2 * B + B * A * 2 + 3 * B)   # reads + dz x2, y, q_sel x2
    actor = 4 * (B * A * (3 + noise) + B + B * A + B)                # reads + dz, weight
    return dict(critic_head=critic, actor_head=actor)


def build_fused(cfg, dev):
    import torch

    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import FullyConnectedActor, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import DiscreteCRRTrainer

    torch.manual_seed(0)
    S, A, sizes = cfg["S"], cfg["A"], cfg["sizes"]
    acts = ["relu"] * len(sizes)
    actor = FullyConnectedActor(S, A, sizes, acts, exploration_variance=cfg["noise"]).to(dev)
    q1 = FullyConnectedDQN(S, A, sizes, acts).to(dev)
    q2 = FullyConnectedDQN(S, A, sizes, acts).to(dev)
    return DiscreteCRRTrainer(
        actor_network=actor, actor_network_target=actor.get_target_network(), q1_network=q1,
        q1_network_target=q1.get_target_network(), reward_network=None, q2_network=q2,
        q2_network_target=q2.get_target_network(),
        evaluation=EvaluationParameters(calc_cpe_in_training=False),
        rl=RLParameters(gamma=cfg["gamma"], target_update_rate=cfg["tau"]),
        q_network_optimizer=Optimizer__Union.default(lr=LR),
        actor_network_optimizer=Optimizer__Union.default(lr=LR),
        actions=[str(i) for i in range(A)]).to(dev)


class EagerCRR:
    """The same update in eager torch, written for this measurement."""

    def __init__(self, fused, cfg, dev):
        import copy

        import torch

        def seq(net, last):
            layers = []
            n = len(net.fc.dnn)
            for i, s in enumerate(net.fc.dnn):
                lin = torch.nn.Linear(s[0].in_features, s[0].out_features)
                with torch.no_grad():
                    lin.weight.copy_(s[0].weight)
                    lin.bias.copy_(s[0].bias)
                layers += [lin, torch.nn.ReLU() if i < n - 1 else last()]
            return torch.nn.Sequential(*layers).to(dev)

        self.cfg = cfg
        self.actor = seq(fused.actor_network, torch.nn.Tanh)
        self.q1 = seq(fused.q1_network, torch.nn.Identity)
        self.q2 = seq(fused.q2_network, torch.nn.Identity)
        self.targets = [copy.deepcopy(m) for m in (self.actor, self.q1, self.q2)]
        self.opts = [torch.optim.Adam(m.parameters(), lr=LR, capturable=True)
                     for m in (self.q1, self.q2, self.actor)]

    def _logits(self, net, x):
        import torch

        out = net(x)
        scale = self.cfg["noise"]
        if scale is None:
            return out
        return (out + torch.randn_like(out) * scale).clamp(-1.0, 1.0)

    def step(self, b):
        import torch
        import torch.nn.functional as F
        from torch.distributions import Categorical

        gamma, tau = self.cfg["gamma"], self.cfg["tau"]
        at, q1t, q2t = self.targets
        with torch.no_grad():
            p = Categorical(logits=self._logits(self.actor, b["next_state"]), validate_args=False).probs
            v = torch.min((q1t(b["next_state"]) * p).sum(1, keepdim=True),
                          (q2t(b["next_state"]) * p).sum(1, keepdim=True))
            y = b["reward"] + gamma * v * b["not_terminal"]
        losses = []
        for q, opt in ((self.q1, self.opts[0]), (self.q2, self.opts[1])):
            loss = F.mse_loss((q(b["state"]) * b["action"]).sum(1, keepdim=True), y)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.detach())
        with torch.no_grad():
            all_q = self.q1(b["state"])
        dist = Categorical(logits=self._logits(self.actor, b["state"]), validate_args=False)
        values = (all_q * dist.probs).sum(1, keepdim=True)
        adv = ((all_q - values) * b["action"]).sum(1, keepdim=True)
        weight = torch.clamp(adv.exp(), 0, 20.0).detach()
        log_pi = dist.log_prob(b["action"].argmax(1)).unsqueeze(1)
        aloss = (-log_pi * weight).mean()
        self.opts[2].zero_grad(set_to_none=True)
        aloss.backward()
        self.opts[2].step()
        with torch.no_grad():
            for t, s in zip(self.targets, (self.actor, self.q1, self.q2)):
                tp, sp = list(t.parameters()), list(s.parameters())
                torch._foreach_mul_(tp, 1.0 - tau)
                torch._foreach_add_(tp, sp, alpha=tau)
        return losses[0]


def make_batch(cfg, dev):
    import torch

    from reagent_b200.core import types as rlt

    g = torch.Generator().manual_seed(1)
    B, S, A = cfg["B"], cfg["S"], cfg["A"]
    d = dict(state=torch.randn(B, S, generator=g), next_state=torch.randn(B, S, generator=g),
             reward=torch.randn(B, 1, generator=g),
             not_terminal=(torch.rand(B, 1, generator=g) > 0.05).float(),
             action=torch.nn.functional.one_hot(torch.randint(A, (B,), generator=g), A).float(),
             prob=torch.rand(B, 1, generator=g) * 0.8 + 0.1)
    d = {k: v.to(dev) for k, v in d.items()}
    batch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(d["state"]), next_state=rlt.FeatureData(d["next_state"]),
        reward=d["reward"], time_diff=torch.ones_like(d["reward"]), step=None,
        not_terminal=d["not_terminal"], action=d["action"],
        next_action=torch.zeros_like(d["action"]),
        possible_actions_mask=torch.ones_like(d["action"]),
        possible_next_actions_mask=torch.ones_like(d["action"]),
        extras=rlt.ExtraData(action_probability=d["prob"]))
    return d, batch


def capture(fn, calls, warmup=5):
    """A CUDA graph of `calls` consecutive calls of fn, captured after `warmup` eager calls."""
    import torch

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    return g


def replay_us(g, calls):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls


def alternate(graphs, calls, reps):
    for g in graphs.values():  # one untimed replay each
        replay_us(g, calls)
    runs = {k: [] for k in graphs}
    for rep in range(reps):
        order = list(graphs) if rep % 2 == 0 else list(graphs)[::-1]
        for k in order:
            runs[k].append(replay_us(graphs[k], calls))
    return {k: dict(median=statistics.median(v), min=min(v), max=max(v), all=v)
            for k, v in runs.items()}


def head_calls(trainer, batch):
    """Closures launching each head alone on the trainer's workspace (left by one update)."""
    from reagent_b200 import _lib

    ws, lib, B, A = trainer._ws, _lib.lib(), batch.action.shape[0], trainer.num_actions
    keep = [batch.reward.reshape(-1).contiguous(), batch.not_terminal.reshape(-1).contiguous(),
            batch.extras.action_probability.reshape(-1).contiguous()]
    c = _lib.CrrCriticArgsT()
    c.batch, c.num_actions = B, A
    c.actor_next, c.q1_target_next = ws["actor_next"].data_ptr(), ws["q1t_next"].data_ptr()
    c.q2_target_next, c.q1, c.q2 = (ws["q2t_next"].data_ptr(), ws["q1_out"].data_ptr(),
                                    ws["q2_out"].data_ptr())
    c.action, c.reward, c.not_terminal = batch.action.data_ptr(), keep[0].data_ptr(), keep[1].data_ptr()
    c.gamma = float(trainer.gamma)
    c.td_target, c.q1_selected, c.q2_selected = (ws["td_target"].data_ptr(), ws["q1_sel"].data_ptr(),
                                                 ws["q2_sel"].data_ptr())
    c.dz_q1, c.dz_q2 = ws["q1"].dz[-1].data_ptr(), ws["q2"].dz[-1].data_ptr()
    c.loss_partials, c.loss = ws["critic_partials"].data_ptr(), ws["critic_loss"].data_ptr()
    c.tile_counter = ws["counter"][0:1].data_ptr()
    a = _lib.CrrActorArgsT()
    a.batch, a.num_actions = B, A
    a.actor_out, a.q1, a.action = (ws["actor_out"].data_ptr(), ws["q1_out"].data_ptr(),
                                   batch.action.data_ptr())
    a.action_probability = keep[2].data_ptr()
    a.inv_beta, a.max_weight, a.entropy_coeff, a.clip_limit = 1.0, 20.0, 0.0, 10.0
    a.action_activation = _lib.ACT["tanh"]
    a.weight, a.dz = ws["weight"].data_ptr(), ws["actor"].dz[-1].data_ptr()
    a.loss_partials, a.loss = ws["actor_partials"].data_ptr(), ws["actor_loss"].data_ptr()
    a.tile_counter = ws["counter"][1:2].data_ptr()

    def critic():
        _lib.check(lib.rb200_crr_critic_head(c, _lib.cur_stream()), "rb200_crr_critic_head")

    def actor():
        _lib.check(lib.rb200_crr_actor_head(a, _lib.cur_stream()), "rb200_crr_actor_head")

    return {"critic_head": critic, "actor_head": actor}, keep


def time_online(cfg, dev, steps):
    import numpy as np
    import torch

    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep

    S, A, B = cfg["S"], cfg["A"], cfg["B"]
    rng = np.random.RandomState(0)
    n = 8192
    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=16384, batch_size=B, device=dev)
    rb.add_batch(observation=rng.standard_normal((n, S)).astype(np.float32),
                 action=rng.randint(0, A, n).astype(np.int64),
                 reward=rng.standard_normal(n).astype(np.float32),
                 terminal=rng.rand(n) < 0.02, priority=rng.uniform(0.1, 10.0, n))
    fused = FusedDqnStep(build_fused(cfg, dev), rb, B, rng="device", online=True)
    tr = dict(observation=rng.standard_normal(S).astype(np.float32), action=1, reward=0.5,
              terminal=False, priority=1.0)
    for _ in range(20):
        fused.step(tr)
    out = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fused.step(tr)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) / steps * 1e6)
    fused.dr.raise_if_failed()
    return dict(median=statistics.median(out), all=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--steps", type=int, default=300)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_crr.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card_info()
    results = {}
    for name, cfg in SHAPES.items():
        d, batch = make_batch(cfg, dev)
        fused = build_fused(cfg, dev)
        eager = EagerCRR(fused, cfg, dev)
        first = dict(fused=float(fused.train_batch(batch, 0)[0][0]), eager=float(eager.step(d)))
        graphs = {"fused": capture(lambda: fused.train_batch(batch, 0), args.calls),
                  "eager": capture(lambda: eager.step(d), args.calls)}
        per_update = alternate(graphs, args.calls, args.reps)
        calls, keep = head_calls(fused, batch)
        heads = alternate({k: capture(fn, args.calls) for k, fn in calls.items()}, args.calls,
                          args.reps)
        results[name] = dict(
            config=dict(cfg, lr=LR, acts="relu", twin=True), first_q1_loss=first,
            per_update_us=per_update,
            eager_over_fused=per_update["eager"]["median"] / per_update["fused"]["median"],
            head_us=heads, head_algorithmic_bytes=algorithmic_bytes(cfg),
            online_step_us=time_online(cfg, dev, args.steps))
        del graphs, keep
    res = {
        "what": "DiscreteCRRTrainer.train_batch vs the same update in eager torch, the CRR loss "
                "heads alone, and the captured online FusedDqnStep step",
        "card": info,
        "method": (f"CUDA events around one replay of a CUDA graph of {args.calls} consecutive "
                   f"calls, captured after warm-up; medians of {args.reps} runs, variants "
                   f"alternating; online step: host clock over {args.steps} steps ending in a "
                   "synchronise, 3 repetitions"),
        "results": results,
    }
    smi = list(info["nvidia_smi"].values())[0].split(",")
    model = re.search(r"\b([a-z]+\d+)\b", smi[0].lower()) if len(smi) == 3 else None  # "h100"
    card = model.group(1) if model else "gpu"
    limit = re.sub(r"[^0-9.]", "", smi[1]).split(".")[0] if len(smi) == 3 else "unknown"
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"time_crr_{card}_{limit}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    print("wrote", path)


if __name__ == "__main__":
    main()
