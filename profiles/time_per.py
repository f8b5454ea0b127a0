"""Cost of prioritized experience replay (FusedDqnStep(per=...)) at config-2 shapes (B 4096,
replay capacity 2^20, q-network 128-256-128-16 relu, Huber, double-Q).

PER adds three things to every update of FusedDqnStep(rng="device", online=True): the
importance-weight kernel before K2, the weighted K2 instantiation, and the priority write-back
(the ordered batched SumTree.set) after the update.  This script times, in one process:
  * FusedDqnStep.step() per update with and without `per`, alternating the two variants;
  * the batched SumTree.set alone at n = 4096 on a 2^20-leaf tree, against the one-warp
    sequential kernel it replaced (compiled here from its source below into a temporary
    directory), with CUDA events over many launches;
and records the card's name, power limit and maximum SM clock read in the same run.

    python profiles/time_per.py --out DIR [--reps 11] [--steps 200]

Writes DIR/time_per.json and prints the same JSON.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CAPACITY = 1 << 20

# the sequential one-warp SumTree.set kernel that rb200_sumtree_set_device ran before the
# ordered batched update: lane l owns level l of the root path, one set after another
OLD_KERNEL = r"""
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ void tree_set_warp(double* tree, int depth, long long leaf, double value,
                                              double* max_recorded, int lane) {
  double delta = 0.0;
  if (lane == depth) {
    delta = value - tree[((1ll << depth) - 1) + leaf];
    if (max_recorded && value > *max_recorded) *max_recorded = value;
  }
  delta = __shfl_sync(0xffffffffu, delta, depth);
  if (lane <= depth) {
    double* p = tree + ((1ll << lane) - 1) + (leaf >> (depth - lane));
    *p = __dadd_rn(*p, delta);
  }
  __syncwarp();
}
__global__ void sumtree_set_kernel(double* tree, int depth, const long long* idx, const double* val,
                                   int n, double* max_recorded, int* status) {
  const int lane = threadIdx.x;
  for (int i = 0; i < n; ++i) {
    const double v = val[i];
    if (v < 0.0) { if (lane == 0 && status) status[0] = 2; return; }
    tree_set_warp(tree, depth, idx[i], v, max_recorded, lane);
  }
}
extern "C" int old_sumtree_set(double* tree, int depth, const int64_t* idx, const double* val,
                               int n, double* max_recorded, int* status, void* stream) {
  sumtree_set_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(tree, depth, (const long long*)idx, val,
                                                         n, max_recorded, status);
  return (int)cudaGetLastError();
}
"""


def card_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    import torch

    return {"torch_device_name": torch.cuda.get_device_name(0), "nvidia_smi": {q: out}}


def build(cfg, dev, per):
    import bench
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAPACITY, batch_size=cfg["B"],
                                 device=dev)
    rb.add_batch(**bench.synth_stream(CAPACITY, 0, cfg))
    t = bench.build_trainer(cfg, dev, seed=0)
    return FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=per)


def transitions(cfg, n):
    import bench

    st = bench.synth_stream(n, 1, cfg)
    return [{k: v[i] for k, v in st.items()} for i in range(n)]


def time_steps(fused, trs, steps, k0):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        lh = fused.step(trs[(k0 + i) % len(trs)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps, float(lh[0])


def time_launches(fn, n):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        fn()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n  # microseconds per launch


def old_kernel_lib(tmp):
    src = os.path.join(tmp, "old_sumtree.cu")
    so = os.path.join(tmp, "libold_sumtree.so")
    with open(src, "w") as f:
        f.write(OLD_KERNEL)
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared",
                    "-Xcompiler", "-fPIC", src, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    lib.old_sumtree_set.argtypes = [vp, ctypes.c_int, vp, vp, ctypes.c_int, vp, vp, vp]
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for time_per.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedUpdate

    if not torch.cuda.is_available():
        raise SystemExit("time_per.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = dict(bench.CONFIGS[2])
    info = card_info()
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=100_000, eps=1e-6)
    variants = {"plain": build(cfg, dev, None), "per": build(cfg, dev, per)}
    trs = transitions(cfg, 1000)
    for fused in variants.values():
        time_steps(fused, trs, args.warmup, 0)
    per_update = {k: [] for k in variants}
    last_loss = {}
    for rep in range(args.reps):
        order = list(variants) if rep % 2 == 0 else list(variants)[::-1]
        for k in order:
            dt, last_loss[k] = time_steps(variants[k], trs, args.steps, rep * args.steps)
            per_update[k].append(dt * 1e6)
    for fused in variants.values():
        fused.dr.raise_if_failed()

    # the tree update alone, n = 4096 sets with a batch's duplicate pattern, 2^20 leaves
    B = cfg["B"]
    depth = 20
    rng = np.random.RandomState(0)
    tree = torch.from_numpy(np.zeros((1 << (depth + 1)) - 1)).to(dev)
    idx = torch.from_numpy(rng.randint(0, CAPACITY, B).astype(np.int64)).to(dev)
    val = torch.from_numpy(rng.uniform(0.1, 10.0, B)).to(dev)
    mx = torch.zeros(1, dtype=torch.float64, device=dev)
    st = torch.zeros(2, dtype=torch.int32, device=dev)
    lib, stream = _lib.lib(), _lib.cur_stream()
    with tempfile.TemporaryDirectory() as tmp:
        old = old_kernel_lib(tmp)

        def new_update():
            _lib.check(lib.rb200_sumtree_set_device(tree.data_ptr(), depth, idx.data_ptr(),
                                                    val.data_ptr(), B, mx.data_ptr(),
                                                    st.data_ptr(), stream))

        def old_update():
            assert old.old_sumtree_set(tree.data_ptr(), depth, idx.data_ptr(), val.data_ptr(), B,
                                       mx.data_ptr(), st.data_ptr(), stream) == 0

        kern = {}
        for rep in range(3):
            for name, fn in (("batched_sumtree_set", new_update), ("one_warp_sumtree_set", old_update)):
                kern.setdefault(name, []).append(time_launches(fn, args.launches))
        # both give the same tree from the same start
        tree.zero_(); mx.zero_()
        new_update()
        a = tree.clone()
        tree.zero_(); mx.zero_()
        old_update()
        same = bool(torch.equal(a, tree))

    med = {k: statistics.median(v) for k, v in per_update.items()}
    kmed = {k: statistics.median(v) for k, v in kern.items()}
    res = {
        "what": ("FusedDqnStep(rng='device', online=True).step() per update, config-2 shapes, "
                 "with and without per; the batched SumTree.set against the one-warp kernel"),
        "card": info,
        "config": dict(B=B, S=cfg["S"], A=cfg["A"], sizes=cfg["sizes"],
                       replay_capacity=CAPACITY, per=dict(alpha=per.alpha, beta0=per.beta0,
                                                          beta_updates=per.beta_updates,
                                                          eps=per.eps)),
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps; tree "
                   f"updates: CUDA events over {args.launches} back-to-back launches, 3 "
                   f"repetitions, n = {B} sets on a 2^{depth}-leaf tree"),
        "per_update_us": {k: dict(median=med[k], min=min(v), max=max(v), all=v)
                          for k, v in per_update.items()},
        "per_overhead_us_median": med["per"] - med["plain"],
        "per_overhead_frac_median": med["per"] / med["plain"] - 1,
        "tree_update_us": {k: dict(median=kmed[k], all=v) for k, v in kern.items()},
        "tree_update_speedup_median": kmed["one_warp_sumtree_set"] / kmed["batched_sumtree_set"],
        "tree_update_results_identical": same,
        "last_loss": last_loss,
    }
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_per.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
