"""Time Seq2Reward's fused update and plan against the same computations in eager torch on the
same GPU (cuDNN nn.LSTM, the reference's formulas, torch.optim.Adam(foreach=True)).

Shapes: the reference's seq2reward_test.yaml (S 2, A 2, T 6, B 1024, H 64, L 2, multi_steps 6)
and, for get_Q, a heavier one (S 2, A 3, k 6, H 128, L 2, B 256).  Seeded, untrained networks.
Alternating the variants in one process, medians over repetitions:
  * train:     Seq2RewardTrainer.train_batch against the reference's get_mse_loss +
               get_step_entropy_loss, backward and two Adam steps;
  * get_q:     get_Q (the prefix-tree plan) against the reference's get_Q on the expanded batch;
  * q_all:     every horizon 1..k from one plan against get_Q once per length;
  * compress:  CompressModelTrainer.train_batch against the reference's get_loss, backward, Adam;
  * kernels:   each rb200_seq2reward_* launch alone, CUDA events around back-to-back launches.
The card's name, power limit and maximum SM clock are read in the same run.

    python profiles/time_seq2reward.py --out DIR [--reps 5] [--steps 50]

Writes DIR/time_seq2reward_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import alternate, card_info, cuda_device, launch_us, write_result  # noqa: E402

TRAIN = dict(S=2, A=2, T=6, B=1024, H=64, L=2, k=6, lr=0.005)
PLANS = {"yaml_b1024_a2_k6_h64": dict(S=2, A=2, k=6, H=64, L=2, B=1024),
         "heavy_b256_a3_k6_h128": dict(S=2, A=3, k=6, H=128, L=2, B=256)}


def _batch(c, dev, seed=0):
    import torch

    from reagent_b200.core import types as rlt

    g = torch.Generator().manual_seed(seed)
    T, B, S, A = c["T"], c["B"], c["S"], c["A"]
    state = torch.randn(T, B, S, generator=g)
    action = torch.nn.functional.one_hot(torch.randint(0, A, (T, B), generator=g), A).float()
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(state.to(dev)), next_state=rlt.FeatureData(state.to(dev)),
        action=rlt.FeatureData(action.to(dev)), reward=torch.randn(T, B, generator=g).to(dev),
        not_terminal=torch.ones(T, B, device=dev), time_diff=None, step=None,
        valid_step=torch.randint(1, c["k"] + 1, (B, 1), generator=g).to(dev))


class Eager(object):
    """The reference's Seq2RewardNetwork / step network / compress network in plain torch."""

    def __init__(self, S, A, H, L, k, dev, step_size=64, compress=(256, 128)):
        import torch
        import torch.nn as nn

        self.rnn = nn.LSTM(A, H, L).to(dev)
        self.lstm_linear = nn.Linear(H, 1).to(dev)
        self.map_linear = nn.Linear(S, H).to(dev)
        self.step = nn.Sequential(nn.Linear(S, step_size), nn.ReLU(), nn.Linear(step_size, step_size),
                                  nn.ReLU(), nn.Linear(step_size, k)).to(dev)
        self.comp = nn.Sequential(nn.Linear(S, compress[0]), nn.ReLU(),
                                  nn.Linear(compress[0], compress[1]), nn.ReLU(),
                                  nn.Linear(compress[1], A)).to(dev)
        self.L, self.A, self.k = L, A, k
        self.torch = torch

    def net_params(self):
        return (list(self.rnn.parameters()) + list(self.lstm_linear.parameters())
                + list(self.map_linear.parameters()))

    def forward(self, state0, action, valid=None):
        torch = self.torch
        h0 = self.map_linear(state0.unsqueeze(0).repeat(self.L, 1, 1))
        out, _ = self.rnn(action, (h0, torch.zeros_like(h0)))
        B = action.shape[1]
        sel = out[-1] if valid is None else out[valid - 1, torch.arange(B, device=out.device)]
        return self.lstm_linear(sel)

    def get_q(self, state, permut):
        torch = self.torch
        B = state.shape[0]
        n = permut.shape[1]
        s = state.repeat_interleave(n, dim=0)
        r = self.forward(s, permut.repeat(1, B, 1)).reshape(B, self.A, n // self.A)
        return torch.max(r, dim=2).values


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory of the JSON result")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    dev = cuda_device(__file__)

    import torch
    import torch.nn.functional as F

    from reagent_b200 import _lib
    from reagent_b200.core.parameters import Seq2RewardTrainerParameters
    from reagent_b200.models import FloatFeatureFullyConnected, Seq2RewardNetwork
    from reagent_b200.models.seq2reward_model import run_forward
    from reagent_b200.training import CompressModelTrainer, Seq2RewardTrainer, gen_permutations, get_Q

    torch.backends.cudnn.benchmark = False
    res = {"card": card_info(), "train_shape": TRAIN, "plan_shapes": PLANS, "unit": "us",
           "reps": args.reps, "steps": args.steps}
    n = args.steps

    def timed(fn):
        def run(_name, _rep):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            return launch_us(fn, n, warmup=0)
        return run

    # ---- training step ---------------------------------------------------
    c = TRAIN
    torch.manual_seed(0)
    params = Seq2RewardTrainerParameters(learning_rate=c["lr"], multi_steps=c["k"],
                                         action_names=["0", "1"])
    tr = Seq2RewardTrainer(Seq2RewardNetwork(c["S"], c["A"], c["H"], c["L"]), params).to(dev)
    batch = _batch(c, dev)
    eg = Eager(c["S"], c["A"], c["H"], c["L"], c["k"], dev)
    opt1 = torch.optim.Adam(eg.net_params(), lr=c["lr"], foreach=True)
    opt2 = torch.optim.Adam(eg.step.parameters(), lr=c["lr"], foreach=True)
    T, B = c["T"], c["B"]
    gamma_mask = torch.ones(T, B, device=dev)
    valid = batch.valid_step.flatten()
    s0 = batch.state.float_features[0]

    def eager_train():
        pred = eg.forward(s0, batch.action.float_features, valid)
        tgt = torch.cumsum(batch.reward * gamma_mask, dim=0)[valid - 1, torch.arange(B, device=dev)]
        loss = F.mse_loss(pred, tgt.unsqueeze(1))
        opt1.zero_grad()
        loss.backward()
        opt1.step()
        sl = F.cross_entropy(eg.step(s0), valid - 1)
        opt2.zero_grad()
        sl.backward()
        opt2.step()

    res["train"] = alternate(["fused", "eager"], args.reps, lambda k, r: timed(
        (lambda: tr.train_batch(batch)) if k == "fused" else eager_train)(k, r))

    # ---- get_Q and every horizon ----------------------------------------
    res["get_q"], res["q_all"] = {}, {}
    for name, p in PLANS.items():
        torch.manual_seed(0)
        net = Seq2RewardNetwork(p["S"], p["A"], p["H"], p["L"]).to(dev)
        e = Eager(p["S"], p["A"], p["H"], p["L"], p["k"], dev)
        state = torch.randn(p["B"], p["S"], device=dev)
        perms = {j: gen_permutations(j, p["A"]).to(dev) for j in range(1, p["k"] + 1)}
        permut_cpu = gen_permutations(p["k"], p["A"])
        with torch.no_grad():
            res["get_q"][name] = alternate(["fused", "eager"], args.reps, lambda k, r: timed(
                (lambda: get_Q(net, state, permut_cpu)) if k == "fused"
                else (lambda: e.get_q(state, perms[p["k"]])))(k, r))
            res["q_all"][name] = alternate(["fused", "eager_per_length"], args.reps, lambda k, r: timed(
                (lambda: net.plan(state, p["k"], all_horizons=True)) if k == "fused"
                else (lambda: [e.get_q(state, perms[j]) for j in range(1, p["k"] + 1)]))(k, r))

    # ---- compress --------------------------------------------------------
    torch.manual_seed(1)
    comp = FloatFeatureFullyConnected(c["S"], c["A"], [256, 128], ["relu", "relu"]).to(dev)
    ct = CompressModelTrainer(comp, tr.seq2reward_network, params)
    opt3 = torch.optim.Adam(eg.comp.parameters(), lr=params.compress_model_learning_rate, foreach=True)
    perm_k = gen_permutations(c["k"], c["A"]).to(dev)

    def eager_compress():
        out = eg.comp(s0)
        with torch.no_grad():
            q = eg.get_q(s0, perm_k)
        loss = F.mse_loss(out, q)
        with torch.no_grad():
            torch.mean((q.argmax(1) == out.argmax(1)).float())
        opt3.zero_grad()
        loss.backward()
        opt3.step()

    res["compress"] = alternate(["fused", "eager"], args.reps, lambda k, r: timed(
        (lambda: ct.train_batch(batch)) if k == "fused" else eager_compress)(k, r))

    # ---- each kernel alone ----------------------------------------------
    net = tr.seq2reward_network
    lib, st = _lib.lib(), _lib.cur_stream()
    ws = tr._ws
    splits = lib.rb200_wgrad_splits(T * B)
    # the arguments of the training step's own launches, on its workspace
    run_forward(net, batch.state.float_features, batch.action.float_features, valid, ws,
                reward=batch.reward, gamma=params.gamma, train=True, multi_steps=c["k"])
    a = net.args(T, B)
    a.state, a.action = ws.keep[0].data_ptr(), ws.keep[1].data_ptr()
    a.hs, a.cs, a.acts, a.dy = ws.hs.data_ptr(), ws.cs.data_ptr(), ws.acts.data_ptr(), ws.dy.data_ptr()
    a.dgates, a.dh0 = ws.dgates.data_ptr(), ws.dh0.data_ptr()
    a.splits, a.gpart = splits, net.arena.gpart.data_ptr()
    ct._step(batch, train=True)
    cw = ct._ws
    h = _lib.Seq2rewardCompressArgsT()
    h.batch, h.num_action = B, c["A"]
    h.out, h.q, h.dout = cw["out"].data_ptr(), cw["q"].data_ptr(), cw["net"].dz[-1].data_ptr()
    h.loss_partials, h.tile_counter = cw["loss_partials"].data_ptr(), cw["counter"].data_ptr()
    h.out_loss = cw["loss"].data_ptr()
    kern = {
        "rb200_seq2reward_forward(train)": lambda: run_forward(
            net, batch.state.float_features, batch.action.float_features, valid, ws,
            reward=batch.reward, gamma=params.gamma, train=True, multi_steps=c["k"]),
        "rb200_seq2reward_backward": lambda: lib.rb200_seq2reward_backward(a, st),
        "rb200_seq2reward_wgrad": lambda: lib.rb200_seq2reward_wgrad(a, st),
        "rb200_seq2reward_plan(yaml)": lambda: net.plan(s0, c["k"]),
        "rb200_seq2reward_compress_head": lambda: lib.rb200_seq2reward_compress_head(h, st),
    }
    res["kernels"] = alternate(list(kern), args.reps, lambda k, r: timed(kern[k])(k, r))
    res["note"] = ("kernels: each entry point alone on the training step's workspace; "
                   "rb200_seq2reward_wgrad is its two split-K launches (LSTM and head over T*B "
                   "rows, map_linear over B rows), rb200_seq2reward_plan its memset, k level "
                   "launches and the decode")
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
