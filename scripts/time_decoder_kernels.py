"""Mean kernel time of every decoder kernel in the bench.py mapping step, from torch.profiler (CUDA activities).

Builds the bench.py problem (same synthetic scan, map and decoder seeds: 82.7 k rays, 776 k samples), runs pipelined mapping steps
with the decoder trained and then with it frozen, and prints one JSON line: per kernel the number of calls and the mean time, plus
the card's name, its power limit and the median SM clock sampled during the profiled steps.

    python scripts/time_decoder_kernels.py [--steps 20]

Nothing is written to disk.  Take end-to-end step times from bench.py, not from this run: the profiler slows the host."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

DECODER_KERNELS = ("k_mlp_wg", "k_wgrad_tc", "k_tc_prepare")


def card(index):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(index)],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, power = (f.strip() for f in out.split(","))
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_decoder_kernels.py needs a CUDA device")
    import nerfloam_b200 as nl
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scans, mu, ms, dec = bench.build_problem(nl, 1, dev)
    pts, cos, pose = scans[0]
    h_dirs, h_gt, h_cos = bench.host_rays(pts, cos)
    R = h_dirs.shape[0]
    dirs, gt, cosv = h_dirs.to(dev), h_gt.to(dev), h_cos.to(dev)
    pose6 = nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)).data.detach().reshape(1, 6).to(dev).contiguous()
    eng = nl.engine.SDFEngine(R, R * 20, dev)
    bufs = nl.engine.DecoderBuffers(dec, dev)
    opt = {}

    def step(update_decoder):   # bench.py's pipelined mapping step
        eng.rays_from_poses(pose6, dirs, None)
        eng.forward_backward(ms, bufs, R, bench.CFG, gt, cosv, dir_local=dirs, ray_frame=None, n_frames=1, rng_seed=12345,
                             update_decoder=update_decoder, update_emb=True, update_pose=True, pose6=pose6,
                             defer_wgrad=update_decoder and eng.overlap_wgrad)
        if update_decoder not in opt:   # the gradient buffers exist after the first iteration
            groups = [dict(param=ms.emb, grad=eng.grad_emb, lr=bench.LR[0]), dict(param=pose6[0], grad=eng.pose_grad[0], lr=bench.LR[2])]
            if update_decoder:
                groups += [dict(param=p.data, grad=g, lr=bench.LR[1], side=True) for p, g in zip(bufs.params, bufs.grads)]
            opt[update_decoder] = nl.engine.FusedAdam(groups, ctl=lambda: eng.ctl)
        opt[update_decoder].step(side_stream=eng.deferred_stream() if update_decoder else None)

    eng.begin_call()
    for _ in range(bench.N_SETTLE):
        step(True)
    for _ in range(3):
        step(False)
    eng.join_side()
    torch.cuda.synchronize()
    n_samples = eng.read_stats().n_samples
    clocks = bench.ClockSampler(0)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step(True)
        eng.join_side()
        for _ in range(args.steps):
            step(False)
        torch.cuda.synchronize()
    clk = clocks.stop()
    kernels = {}
    for ev in prof.key_averages():
        name = ev.key
        if not any(k in name for k in DECODER_KERNELS):
            continue
        total_us = getattr(ev, "device_time_total", None)
        if total_us is None:
            total_us = ev.cuda_time_total
        short = name.split("(")[0].replace("void ", "")
        kernels[short] = {"calls": ev.count, "mean_ms": round(total_us / ev.count / 1e3, 4)}
    name, power = card(0)
    print(json.dumps({"gpu": name, "power_limit": power, "sm_clock_median_mhz": clk["sm_mhz"], "clock_reasons": clk["reasons"],
                      "samples": n_samples, "steps": args.steps, "kernels": kernels}))


if __name__ == "__main__":
    main()
