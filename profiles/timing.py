"""What the profile scripts share: the GPU and the card's identity, CUDA-graph capture, event
timing of graph replays and of eager launches, host-clocked step loops, alternating variants,
and the result file.  torch is imported inside the functions, so that a script's --help does
not load it."""
import json
import os
import re
import statistics
import subprocess
import time

SMI_QUERY = "name,power.limit,clocks.max.sm"


def cuda_device(script):
    """cuda:0, made the current device; without a GPU, SystemExit naming `script`."""
    import torch

    if not torch.cuda.is_available():
        raise SystemExit(f"{os.path.basename(script)} measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    return dev


def card_info():
    """The card's name, power limit and maximum SM clock, as nvidia-smi reports them (queried,
    never set), and torch's name for device 0."""
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={SMI_QUERY}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    import torch

    return {"torch_device_name": torch.cuda.get_device_name(0), "nvidia_smi": {SMI_QUERY: out}}


def capture(fn, n, warmup=5):
    """A CUDA graph of `n` consecutive calls of `fn`, captured after `warmup` eager calls on a side
    stream, so that lazy allocations, module loads and shared-memory opt-ins happen outside it."""
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
        for _ in range(n):
            fn()
    return g


def replay_us(g, n):
    """Microseconds per call of a graph `g` of `n` calls: CUDA events around one replay, after one
    untimed replay."""
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def launch_us(fn, n, warmup=10):
    """Microseconds per launch of `n` back-to-back eager calls of `fn` between two CUDA events,
    after `warmup` calls."""
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        fn()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def host_steps(step, n, start=0):
    """(microseconds per step, last loss) of step(i) for i in start .. start + n - 1, host-clocked
    from a synchronise to the synchronise after the last step.  `step` returns its loss tensor;
    the last loss is that tensor's first element."""
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(start, start + n):
        loss = step(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e6, float(loss.reshape(-1)[0])


def summary(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v), all=v)


def alternate(names, reps, run):
    """run(name, rep) for every name, `reps` times: in the given order on even repetitions and
    reversed on odd ones, so that neither end of the order is favoured.  Returns
    {name: summary of what run returned}."""
    names = list(names)
    out = {k: [] for k in names}
    for rep in range(reps):
        for k in (names if rep % 2 == 0 else names[::-1]):
            out[k].append(run(k, rep))
    return {k: summary(v) for k, v in out.items()}


def transitions(cfg, n, seed=1):
    """`n` single transitions (add() keyword arguments) of bench.synth_stream's stream."""
    import bench

    st = bench.synth_stream(n, seed, cfg)
    return [{k: v[i] for k, v in st.items()} for i in range(n)]


def write_result(out_dir, script, res):
    """Writes `res` to out_dir/<script>_<card>_<limit>w.json, e.g. time_crr_h100_700w.json, with
    the card's model and power limit from res["card"] ("gpu" and "unknown" when nvidia-smi did
    not answer), and prints it."""
    smi = res["card"]["nvidia_smi"][SMI_QUERY].split(",")
    model = re.search(r"\b([a-z]+\d+)\b", smi[0].lower()) if len(smi) == 3 else None  # "h100"
    card = model.group(1) if model else "gpu"
    limit = re.sub(r"[^0-9.]", "", smi[1]).split(".")[0] if len(smi) == 3 else "unknown"
    name = os.path.splitext(os.path.basename(script))[0]
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, f"{name}_{card}_{limit}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    print("wrote", path)
