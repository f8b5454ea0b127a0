"""What one SlateQTrainer update costs on the GPU, against the same update in eager torch.  One
process; records the card's name, power limit and maximum SM clock read in the same run.

Modes: SARSA (the RecSim default), max-Q TOP_K, and multi selection (SARSA, normalised by the
next slate size).  For each mode and shape:
  fused     SlateQTrainer.train_batch as shipped;
  eager     the same update written in plain torch: the reference's sequence of ops (the
            target network re-scores the chosen next slate, top-k over every candidate for
            max-Q), autograd, torch.optim.Adam and a Polyak update, on the same GPU.
Each is a host-clocked loop of --iters updates between two synchronisations, after --warmup
updates; the two run alternately, --reps times, and the medians are reported.  Also timed, with
CUDA events over --iters back-to-back launches: rb200_slateq_head alone with the arguments the
trainer builds, and the next-state forward as the trainer runs it (every one of the C
candidates) against scoring only the K slate entries, which is what SARSA needs.

Shapes: the RecSim configurations (B 1024, C 10, slate 3 so K 4, state 20, doc 20,
[64, 64] leaky_relu; the 20 / 20 widths follow interest evolution's 20 topics) and a wide one
(B 4096, C 100, slate 10, state 128, doc 64, [256, 128] relu).

    python profiles/time_slateq.py --out DIR [--reps 7] [--iters 50] [--warmup 10]

Writes DIR/time_slateq_<card>_<limit>w.json and prints the same JSON.
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
    "recsim": dict(B=1024, C=10, slate=3, S=20, D=20, sizes=[64, 64], act="leaky_relu"),
    "wide": dict(B=4096, C=100, slate=10, S=128, D=64, sizes=[256, 128], act="relu"),
}
MODES = {
    "sarsa": dict(maxq=False, single=True, norm="norm_by_current_slate_size"),
    "topk": dict(maxq=True, single=True, norm="norm_by_current_slate_size"),
    "multi": dict(maxq=False, single=False, norm="norm_by_next_slate_size"),
}


def make_batch(shape, seed=1):
    """A SlateQInputMaker-shaped device batch: slate distinct candidates plus the null slot."""
    import torch

    from reagent_b200.core import types as rlt

    B, C, k, S, D = shape["B"], shape["C"], shape["slate"], shape["S"], shape["D"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    null = torch.full((B, 1), k, dtype=torch.int64, device="cuda")

    def slate():
        return torch.cat([torch.rand(B, C, device="cuda", generator=g).argsort(1)[:, :k], null], 1)

    def fd(s):
        return rlt.FeatureData(s, candidate_docs=rlt.DocList(
            torch.randn(B, C, D, device="cuda", generator=g), torch.ones(B, C, device="cuda"),
            torch.rand(B, C, device="cuda", generator=g)))

    click = torch.rand(B, k, device="cuda", generator=g) < 0.3
    return rlt.SlateQInput(
        state=fd(torch.randn(B, S, device="cuda", generator=g)),
        next_state=fd(torch.randn(B, S, device="cuda", generator=g)),
        reward=torch.cat([torch.rand(B, k, device="cuda", generator=g) * click,
                          torch.zeros(B, 1, device="cuda")], 1),
        reward_mask=torch.cat([click, (click.sum(1) == 0).view(B, 1)], 1),
        not_terminal=torch.rand(B, 1, device="cuda", generator=g) >= 0.1,
        time_diff=None, step=None, action=slate(), next_action=slate())


def build_fused(shape, mode):
    import torch

    from reagent_b200.core.parameters import RLParameters, SlateOptParameters
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import SlateQTrainer

    torch.manual_seed(0)
    q = FullyConnectedCritic(shape["S"], shape["D"], shape["sizes"],
                             [shape["act"]] * len(shape["sizes"])).cuda()
    return SlateQTrainer(q, q.get_target_network(), shape["slate"],
                         rl=RLParameters(maxq_learning=mode["maxq"]),
                         optimizer=Optimizer__Union.default(lr=1e-3),
                         slate_opt_parameters=SlateOptParameters() if mode["maxq"] else None,
                         single_selection=mode["single"],
                         next_slate_value_norm_method=mode["norm"]).cuda()


class Eager:
    """The update as plain torch ops on two torch.nn.Sequential networks."""

    def __init__(self, shape, mode):
        import torch

        act = torch.nn.LeakyReLU if shape["act"] == "leaky_relu" else torch.nn.ReLU
        dims = [shape["S"] + shape["D"]] + shape["sizes"] + [1]
        layers = []
        for i in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
            if i < len(dims) - 2:
                layers.append(act())
        torch.manual_seed(0)
        self.q = torch.nn.Sequential(*layers).cuda()
        self.qt = torch.nn.Sequential(*[type(m)() if not isinstance(m, torch.nn.Linear)
                                        else torch.nn.Linear(m.in_features, m.out_features)
                                        for m in layers]).cuda()
        self.qt.load_state_dict(self.q.state_dict())
        self.opt = torch.optim.Adam(self.q.parameters(), lr=1e-3)
        self.mode, self.slate = mode, shape["slate"]
        self.tau, self.gamma = 0.001, 0.9

    def _score(self, net, state, docs):
        import torch

        B, K, D = docs.shape
        x = torch.cat((state.repeat_interleave(K, dim=0), docs.reshape(B * K, D)), dim=1)
        return net(x).view(B, K)

    def step(self, b):
        import torch
        import torch.nn.functional as F

        single = self.mode["single"]

        def value(v, m):
            v = v * m
            return F.softmax(v, dim=1) if single else v

        rows = torch.arange(b.action.shape[0], device="cuda").unsqueeze(1)
        nd = b.next_state.candidate_docs
        with torch.no_grad():
            if self.mode["maxq"]:
                nxt = torch.topk(self._score(self.qt, b.next_state.float_features, nd.float_features)
                                 * value(nd.value, nd.mask), self.slate, dim=1).indices
            else:
                nxt = b.next_action.clone()
            nxt[~b.not_terminal.squeeze(1)] = 0
            nq = (self._score(self.qt, b.next_state.float_features, nd.float_features[rows, nxt])
                  * value(nd.value[rows, nxt], nd.mask[rows, nxt])).sum(1, keepdim=True)
            if not single:
                nq = nq / torch.clamp(nd.mask.sum(1, keepdim=True), max=self.slate)
            target = b.reward + self.gamma * (nq * b.not_terminal.float())
        docs = b.state.candidate_docs.float_features[rows, b.action]
        qv = self._score(self.q, b.state.float_features, docs)
        if single:
            loss = F.mse_loss(qv[b.reward_mask], target[b.reward_mask])
        else:
            loss = F.mse_loss(qv, target)
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        with torch.no_grad():
            torch._foreach_lerp_(list(self.qt.parameters()), list(self.q.parameters()), self.tau)
        return loss.detach()


def head_call(t):
    """A call of rb200_slateq_head with the arguments of the trainer's last update."""
    from reagent_b200 import _lib

    captured = {}
    lib = _lib.lib()
    real = lib.rb200_slateq_head

    class Spy:
        def rb200_slateq_head(self, a, stream):
            captured["a"] = _lib.SlateqArgsT.from_buffer_copy(a)
            return real(a, stream)

        def __getattr__(self, name):
            return getattr(lib, name)

    orig = _lib.lib
    _lib.lib = lambda: Spy()
    try:
        t.train_batch(t._profile_batch)
    finally:
        _lib.lib = orig
    a = captured["a"]
    # the trainer's float copies of the boolean fields are gone after the update: re-made here
    b = t._profile_batch
    keep = [b.reward_mask.float().contiguous(), b.not_terminal.float().reshape(-1).contiguous()]
    a.reward_mask, a.not_terminal = keep[0].data_ptr(), keep[1].data_ptr()
    return lambda: _lib.check(real(a, _lib.cur_stream()), "rb200_slateq_head") or keep


def next_forwards(t, batch, iters):
    """us per next-state forward over all C candidates (as the trainer runs it) and over the K
    slate entries only."""
    import torch

    from reagent_b200.models.arena import run_mlp_tiled

    ns = batch.next_state.float_features.contiguous()
    nd = batch.next_state.candidate_docs.float_features
    B, C, D = nd.shape
    K = batch.next_action.shape[1]
    rows = torch.arange(B, device="cuda").unsqueeze(1)
    all_c = nd.reshape(B * C, D).contiguous()
    slate = nd[rows, batch.next_action].reshape(B * K, D).contiguous()
    arena = t.q_network_target.arena
    o_all = torch.empty(B * C, 1, device="cuda")
    o_k = torch.empty(B * K, 1, device="cuda")
    return {"all_candidates": launch_us(lambda: run_mlp_tiled([arena], ns, all_c, C, [o_all]), iters),
            "slate_only": launch_us(lambda: run_mlp_tiled([arena], ns, slate, K, [o_k]), iters),
            "rows": {"all_candidates": B * C, "slate_only": B * K}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    cuda_device(__file__)
    import torch

    result = {"card": card_info(), "reps": args.reps, "iters": args.iters,
              "unit": "us per update (host clock, synchronised) or per launch (CUDA events), "
                      "median [min, max] over reps", "shapes": {}}
    for sname, shape in SHAPES.items():
        res = {"shape": shape, "modes": {}}
        batch = make_batch(shape)
        for mname, mode in MODES.items():
            fused, eager = build_fused(shape, mode), Eager(shape, mode)
            fused._profile_batch = batch
            steps = {"fused": lambda i: fused.train_batch(batch), "eager": lambda i: eager.step(batch)}
            for fn in steps.values():
                host_steps(fn, args.warmup)
            times = alternate(sorted(steps), args.reps,
                              lambda k, rep: host_steps(steps[k], args.iters)[0])
            r = {k: {s: times[k][s] for s in ("median", "min", "max")} for k in steps}
            r["eager_over_fused"] = r["eager"]["median"] / r["fused"]["median"]
            head = head_call(fused)
            r["head_alone"] = launch_us(head, args.iters)
            res["modes"][mname] = r
            if mname == "sarsa":
                res["next_forward_sarsa"] = next_forwards(fused, batch, args.iters)
            fused.raise_if_failed()
            del fused, eager
            torch.cuda.synchronize()
        result["shapes"][sname] = res
    write_result(args.out, __file__, result)


if __name__ == "__main__":
    main()
