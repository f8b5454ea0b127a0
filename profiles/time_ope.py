"""Time counterfactual policy evaluation: Evaluator.evaluate_post_training on a sorted page with
logged values (A 8, episodes of 1 to 30 steps, one metric), with both bootstrap index streams, at
100 k and 1 M rows; three of its kernels alone with CUDA events; and the numpy restatement
(oracle/ope_oracle.py: DR rows, sequential DR, the MAGIC j-step statistics and the SLSQP
combination) on the host at 100 k rows.  End-to-end figures are host-clocked from a synchronise
to a synchronise, medians of alternating runs.  The card's name, power limit and maximum SM
clock are read in the same run.

    python profiles/time_ope.py --out DIR [--reps 5]

Writes DIR/time_ope_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import alternate, card_info, cuda_device, launch_us, write_result  # noqa: E402

A = 8


def make_page(n, dev, seed=0):
    import torch

    from reagent_b200.evaluation import EvaluationDataPage

    g = torch.Generator(device=dev).manual_seed(seed)
    lens = torch.randint(1, 31, (n // 15 + 1,), generator=g, device=dev)
    lens = lens[: int((torch.cumsum(lens, 0) < n).sum()) + 1]
    n = int(lens.sum())
    mdp = torch.repeat_interleave(torch.arange(lens.numel(), device=dev), lens).reshape(-1, 1)
    seq = (torch.arange(n, device=dev)
           - torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens)).reshape(-1, 1)
    am = torch.nn.functional.one_hot(torch.randint(0, A, (n,), generator=g, device=dev), A).float()
    mr = torch.randn(n, 2 * A, generator=g, device=dev) + 0.5
    qv = torch.randn(n, 2 * A, generator=g, device=dev) + 0.5
    page = EvaluationDataPage(
        mdp_id=mdp, sequence_number=seq,
        logged_propensities=torch.rand(n, 1, generator=g, device=dev) * 0.8 + 0.1,
        logged_rewards=torch.randn(n, 1, generator=g, device=dev) + 0.5, action_mask=am,
        model_propensities=torch.softmax(torch.randn(n, A, generator=g, device=dev), 1),
        model_rewards=mr[:, :A], model_rewards_for_logged_action=(mr[:, :A] * am).sum(1, keepdim=True),
        model_values=qv[:, :A], logged_metrics=torch.randn(n, 1, generator=g, device=dev),
        model_metrics=mr[:, A:], model_metrics_values=qv[:, A:])
    return page.sort().compute_values(0.9)


def host_oracle(page):
    import numpy as np

    from oracle import ope_oracle as O

    h = {k: getattr(page, k).cpu().numpy() for k in (
        "mdp_id", "model_propensities", "model_values", "action_mask", "logged_rewards",
        "logged_propensities", "model_rewards", "model_rewards_for_logged_action")}
    t0 = time.perf_counter()
    O.dr_rows(h["model_propensities"], h["model_rewards"], h["action_mask"], h["logged_rewards"],
              h["model_rewards_for_logged_action"], h["logged_propensities"])
    O.sdr_episodes(h["model_propensities"], h["model_values"], h["action_mask"],
                   h["logged_rewards"], h["logged_propensities"], h["mdp_id"], 0.9)
    _, jr, cov, sub, _ = O.wsdr_stats(h["model_propensities"], h["model_values"], h["action_mask"],
                                      h["logged_rewards"], h["logged_propensities"], h["mdp_id"],
                                      0.9, 25)
    O.magic_point(jr, cov, np.array(sub))
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory of the result JSON")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    dev = cuda_device(__file__)
    import numpy as np
    import torch

    from reagent_b200 import _lib
    from reagent_b200.evaluation import Evaluator
    from reagent_b200.evaluation import _ope

    res = {"card": card_info(), "unit": "ms", "rows": {}, "kernels_us": {}}
    for n in (100_000, 1_000_000):
        page = make_page(n, dev)
        ev = {rng: Evaluator([str(a) for a in range(A)], 0.9, None, metrics_to_score=["m0"], rng=rng)
              for rng in ("numpy", "device")}

        def run(rng, rep):
            np.random.seed(rep)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev[rng].evaluate_post_training(page)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        run("numpy", 0)
        run("device", 0)
        res["rows"][str(page.mdp_id.shape[0])] = {
            "episodes": int(torch.unique(page.mdp_id).numel()),
            "evaluate_post_training": alternate(["numpy", "device"], args.reps, run)}
        if n == 1_000_000:
            N = page.mdp_id.shape[0]
            prop, qv, am = page.model_propensities, page.model_values.contiguous(), page.action_mask
            r, lp = page.logged_rewards.contiguous(), page.logged_propensities.contiguous()
            mr, mrl = page.model_rewards.contiguous(), page.model_rewards_for_logged_action
            out = [torch.empty(N, device=dev) for _ in range(3)]
            ep = _ope.Episodes(page.mdp_id, page.sequence_number)
            epo = [torch.empty(ep.num, device=dev) for _ in range(2)]
            means = torch.empty(1000, device=dev)
            L = _lib.lib()
            st = _lib.cur_stream()
            res["kernels_us"]["rows"] = N
            res["kernels_us"]["rb200_ope_dr_rows"] = launch_us(lambda: L.rb200_ope_dr_rows(
                N, A, prop.data_ptr(), mr.data_ptr(), am.data_ptr(), r.data_ptr(), mrl.data_ptr(),
                lp.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), st), 50)
            res["kernels_us"]["rb200_ope_sdr"] = launch_us(lambda: L.rb200_ope_sdr(
                ep.num, ep.off.data_ptr(), A, prop.data_ptr(), qv.data_ptr(), am.data_ptr(),
                r.data_ptr(), lp.data_ptr(), 0.9, epo[0].data_ptr(), epo[1].data_ptr(), st), 50)
            res["kernels_us"]["rb200_ope_boot_means_device_rng_1000x250000"] = launch_us(
                lambda: L.rb200_ope_boot_means(out[2].data_ptr(), N, None, 1000, N // 4, 1, 0,
                                               means.data_ptr(), st), 20)
            flags = torch.empty(2, dtype=torch.int32, device=dev)
            starts = torch.empty(N, dtype=torch.uint8, device=dev)
            mdp, seq = page.mdp_id.contiguous(), page.sequence_number.contiguous()
            res["kernels_us"]["rb200_ope_episode_marks"] = launch_us(lambda: L.rb200_ope_episode_marks(
                N, mdp.data_ptr(), seq.data_ptr(), starts.data_ptr(), flags.data_ptr(), st), 50)
            disc = ep.step_discounts(0.9)
            vals = torch.empty_like(r)
            res["kernels_us"]["rb200_ope_logged_values"] = launch_us(lambda: L.rb200_ope_logged_values(
                ep.num, ep.off.data_ptr(), disc.data_ptr(), 1, r.data_ptr(), vals.data_ptr(), st), 50)
            w64 = [torch.empty(N, dtype=torch.float64, device=dev) for _ in range(3)]
            res["kernels_us"]["rb200_ope_wsdr_rows_fp64"] = launch_us(lambda: L.rb200_ope_wsdr_rows(
                ep.num, ep.off.data_ptr(), A, 1, prop.data_ptr(), qv.data_ptr(), am.data_ptr(),
                lp.data_ptr(), w64[0].data_ptr(), w64[1].data_ptr(), w64[2].data_ptr(), st), 50)
            q = torch.randn(N, A, device=dev)
            ro, co = torch.randn(N, 2 * A, device=dev), torch.randn(N, 2 * A, device=dev)
            pam = torch.ones(N, A, device=dev)
            boosts = torch.zeros(A, device=dev)
            po = [torch.empty(N, A, device=dev), torch.empty(N, dtype=torch.int64, device=dev)] + \
                [torch.empty(N, device=dev) for _ in range(4)]
            res["kernels_us"]["rb200_ope_page_K1"] = launch_us(lambda: L.rb200_ope_page(
                N, A, 1, q.data_ptr(), ro.data_ptr(), co.data_ptr(), pam.data_ptr(), am.data_ptr(),
                r.data_ptr(), boosts.data_ptr(), 1.0, po[2].data_ptr(), po[0].data_ptr(),
                po[1].data_ptr(), po[3].data_ptr(), po[4].data_ptr(), po[5].data_ptr(), st), 50)
            ret = torch.randn(25, ep.num, dtype=torch.float64, device=dev)
            cov = torch.empty(25, 25, dtype=torch.float64, device=dev)
            res["kernels_us"]["rb200_ope_cov_25"] = launch_us(lambda: L.rb200_ope_cov(
                ret.data_ptr(), 25, ep.num, cov.data_ptr(), st), 50)
            res["kernels_us"]["not_measured"] = ["rb200_ope_seg_sum", "rb200_ope_wsdr_returns"]
        if n == 100_000:
            res["host_oracle_100k_ms"] = [host_oracle(page) for _ in range(3)]
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
