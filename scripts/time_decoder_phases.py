"""Where the decoder training kernel's time goes: cycle shares of k_mlp_wg's phases in the bench.py mapping step.

Compiles a copy of the library with -DNL_TC_STAMPS into nerf-loam_b200/_stamps/ (the library bench.py loads is not touched), loads
that copy, builds the bench.py problem (82.7 k rays, 776 k samples), runs pipelined mapping steps with the decoder trained and then
with it frozen, and prints one JSON line: per warpgroup and step kind the share of thread 0's cycles spent in each phase, plus the
card's name, its power limit and the median SM clock sampled during the steps.

    python scripts/time_decoder_phases.py [--steps 20] [--build-only]

Phases (thread 0 of each warpgroup, clock64() between stamps; csrc/mlp_tc.cu, StampPhase):
  ring_wait   acquire: waiting for a weight-ring slot to fill (and, in warpgroup 0, thread 0 issuing the copies)
  a_build     forming the A fragments of a GEMM (tf32 hi / lo splits, or the 0/1 mask words)
  wgmma_wait  wgmma.wait_group and the slot's release
  epi1 / epi2 layer-1 / layer-2 epilogues (bias, ReLU, masks, output-layer sums)
  loss        sdf, loss terms and d loss / d sdf
  wgrad       activation staging for the bulk copies and gW0 / gb0
  rest        everything else: wgmma issue, dh1 formation, d feats stores, tile and kernel set-up
The stamps add a few instructions per phase to warpgroup thread 0 only; the kernel time they report is a little above the plain
build's."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
STAMPS_DIR = os.path.join(ROOT, "nerf-loam_b200", "_stamps")
PHASES = ("ring_wait", "a_build", "wgmma_wait", "epi1", "epi2", "loss", "wgrad", "rest")


def build_stamped():
    import importlib
    b = importlib.import_module("nerf-loam_b200.build")
    return b.build(defines=("NL_TC_STAMPS",), out_dir=STAMPS_DIR)


def shares(raw):
    out = {}
    for wg in range(2):
        row = raw[wg * len(PHASES):(wg + 1) * len(PHASES)]
        tot = sum(row)
        out["wg%d" % wg] = {"cycles": tot, **{ph: round(v / tot, 4) if tot else 0.0 for ph, v in zip(PHASES, row)}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--build-only", action="store_true", help="compile the stamped library and exit")
    args = ap.parse_args()
    lib_path = build_stamped()
    if args.build_only:
        print(lib_path)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_decoder_phases.py needs a CUDA device")
    import bench
    import nerfloam_b200 as nl
    from scripts.time_decoder_kernels import card
    nl._capi.LIB_PATH = lib_path
    L = nl._capi.lib()
    L.nl_mlp_tc_stamps.restype = C.c_int
    L.nl_mlp_tc_stamps.argtypes = [C.c_void_p]
    raw = (C.c_ulonglong * (2 * len(PHASES)))()

    def read():
        torch.cuda.synchronize()
        nl._capi.check(L.nl_mlp_tc_stamps(C.addressof(raw)), "nl_mlp_tc_stamps")
        return list(raw)

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
        if update_decoder not in opt:
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
    read()                      # drop the warm-up's counts
    n_samples = eng.read_stats().n_samples
    clocks = bench.ClockSampler(0)
    for _ in range(args.steps):
        step(True)
    eng.join_side()
    trained = shares(read())
    for _ in range(args.steps):
        step(False)
    frozen = shares(read())
    clk = clocks.stop()
    name, power = card(0)
    print(json.dumps({"gpu": name, "power_limit": power, "sm_clock_median_mhz": clk["sm_mhz"], "clock_reasons": clk["reasons"],
                      "samples": n_samples, "steps": args.steps, "decoder_trained": trained, "decoder_frozen": frozen}))


if __name__ == "__main__":
    main()
