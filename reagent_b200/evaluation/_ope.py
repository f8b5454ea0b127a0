"""Launch plumbing of the evaluation kernels (csrc/rb200_ope.cu): episode offsets, fixed-order
segment sums and the bootstrap sample means."""
import numpy as np
import torch

from .. import _lib

MAX_ROWS = 2 ** 31 - 1


def _call(name, *args):
    _lib.check(getattr(_lib.lib(), name)(*args, _lib.cur_stream()), name)


def require_cuda(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise _lib.Rb200Error(f"{what} must be a CUDA tensor (the evaluation kernels run on the GPU)")
    return t


def f32(t: torch.Tensor, what: str) -> torch.Tensor:
    return require_cuda(t, what).float().contiguous()


def check_ids(mdp_id, sequence_number):
    """mdp_id and sequence_number are int64 (N, 1) device tensors with N < 2**31."""
    for name, t in (("mdp_id", mdp_id), ("sequence_number", sequence_number)):
        require_cuda(t, name)
        if t.dtype != torch.int64 or t.dim() != 2 or t.shape[1] != 1:
            raise ValueError(f"{name} must be an int64 tensor of shape (N, 1), got "
                             f"{t.dtype} {tuple(t.shape)}")
    if mdp_id.shape[0] != sequence_number.shape[0]:
        raise ValueError("mdp_id and sequence_number have different lengths")
    if not 0 < mdp_id.shape[0] <= MAX_ROWS:
        raise ValueError(f"an evaluation page holds 1 to {MAX_ROWS} rows, got {mdp_id.shape[0]}")


class Episodes:
    """Runs of equal mdp_id: offsets [E+1] (int32, device), plus validate()'s two checks:
    the first row whose sequence_number does not increase inside its run (-1 if none) and the
    number of runs."""

    def __init__(self, mdp_id, sequence_number):
        check_ids(mdp_id, sequence_number)
        n = mdp_id.shape[0]
        dev = mdp_id.device
        mdp, seq = mdp_id.contiguous(), sequence_number.contiguous()
        is_start = torch.empty(n, dtype=torch.uint8, device=dev)
        flags = torch.empty(2, dtype=torch.int32, device=dev)
        _call("rb200_ope_episode_marks", n, mdp.data_ptr(), seq.data_ptr(), is_start.data_ptr(),
              flags.data_ptr())
        starts = torch.nonzero(is_start).reshape(-1)
        self.off = torch.cat((starts, torch.tensor([n], device=dev))).to(torch.int32)
        self.num = int(starts.numel())
        bad, runs = flags.tolist()
        self.first_bad_row = -1 if bad == n else bad
        self.runs = runs
        self.n = n
        self.seq = seq

    def lengths(self) -> torch.Tensor:
        return (self.off[1:] - self.off[:-1]).long()

    def step_discounts(self, gamma: float) -> torch.Tensor:
        """[N] float32: row r holds float(math.pow(gamma, seq[r+1] - seq[r])), the factor
        compute_values_for_mdps applies; pow runs on the host (libm, as the reference's
        math.pow) once per distinct gap."""
        seq = self.seq.reshape(-1)
        gaps, where = torch.unique(seq[1:] - seq[:-1], return_inverse=True)
        table = np.power(float(gamma), gaps.cpu().numpy().astype(np.float64)).astype(np.float32)
        disc = torch.ones(self.n, dtype=torch.float32, device=seq.device)
        disc[:-1] = torch.from_numpy(table).to(seq.device)[where]
        return disc


def episodes(edp) -> Episodes:
    """The Episodes of a page, built once per page and shared by the pages _replace derives
    from it without changing mdp_id or sequence_number."""
    ep = edp.__dict__.get("_episodes")
    if ep is None:
        ep = Episodes(edp.mdp_id, edp.sequence_number)
        edp.__dict__["_episodes"] = ep
    return ep


def seg_sum(x: torch.Tensor, seg_off: torch.Tensor, perm=None) -> torch.Tensor:
    """out[s] = sum of x[perm[i]] over i in [seg_off[s], seg_off[s+1]), in a fixed order
    (fp64 accumulation, stored in x's dtype)."""
    nseg = seg_off.numel() - 1
    out = torch.empty(nseg, dtype=x.dtype, device=x.device)
    seg_off = seg_off.to(torch.int64).contiguous()
    _call("rb200_ope_seg_sum", int(x.dtype == torch.float64), x.data_ptr(),
          None if perm is None else perm.data_ptr(), seg_off.data_ptr(), nseg, out.data_ptr())
    return out


def mean(x: torch.Tensor) -> float:
    """float(torch.mean(x)) of a device vector, as one fixed-order sum."""
    x = x.reshape(-1).contiguous()
    s = seg_sum(x, torch.tensor([0, x.numel()], device=x.device))
    return float(s.double().item()) / x.numel()


# index draws uploaded per chunk: at most this many int32 indices on the host at once
_IDX_CHUNK = 1 << 22


def bootstrap_means(data: torch.Tensor, sample_size: int, num_samples: int, rng: str) -> np.ndarray:
    """The `num_samples` bootstrap sample means of bootstrapped_std_error_of_mean, float64.

    rng="numpy": sample i is np.random.choice(data, sample_size, replace=True), which draws
    np.random.randint(0, len(data), sample_size) from the global stream; the draws are made in
    the reference's order and uploaded in int32 chunks.  rng="device": the kernel draws from
    Philox with the seed and offset of torch's CUDA generator, which it then advances."""
    if rng not in ("numpy", "device"):
        raise ValueError(f"rng must be 'numpy' or 'device', got {rng!r}")
    data = f32(data, "bootstrap data").reshape(-1)
    n = data.numel()
    means = torch.empty(num_samples, dtype=torch.float64, device=data.device)
    if sample_size <= 0:
        # np.mean of an empty sample is nan (with numpy's RuntimeWarning)
        if rng == "numpy":
            for _ in range(num_samples):
                np.random.randint(0, n, sample_size)
        return np.full(num_samples, np.nan)
    if rng == "numpy":
        per = max(1, _IDX_CHUNK // sample_size)
        for s0 in range(0, num_samples, per):
            cnt = min(per, num_samples - s0)
            idx = np.empty((cnt, sample_size), dtype=np.int32)
            for i in range(cnt):
                idx[i] = np.random.randint(0, n, sample_size)
            dev_idx = torch.from_numpy(idx).to(data.device)
            _call("rb200_ope_boot_means", data.data_ptr(), n, dev_idx.data_ptr(), cnt, sample_size,
                  0, 0, means[s0:].data_ptr())
    else:
        gen = torch.cuda.default_generators[data.device.index or 0]
        seed, offset = gen.initial_seed(), gen.get_offset()
        per_thread = 2 * ((sample_size + 255) // 256)
        gen.set_offset(offset + ((per_thread + 3) // 4) * 4)
        seed = seed - (1 << 64) if seed >= (1 << 63) else seed  # the ABI's int64_t carries the bits
        _call("rb200_ope_boot_means", data.data_ptr(), n, None, num_samples, sample_size,
              seed, offset, means.data_ptr())
    return means.cpu().numpy()
