"""localise.Localiser's recovery of lost scans on the GPU, against a street map saved by slam.NeRFLOAM (test_gpu_localise.py's map and
second pass: shifted 0.5 m and turned 10 degrees): a gap of dropped scans, a restart metres away and turned beyond the local lattice,
scans the map cannot explain inserted mid-drive, a healthy drive that recovery must leave alone, the map's buffers after all of them,
and scripts/localise.py --recover.  Bounds are test_gpu_localise.py's: 0.10 m and 0.01 (Frobenius)."""
import json
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_gpu_localise import MAX_DR, MAX_DT, N_MAP, ROOT, SHIFT, TURN, MemoryStream, _buffers, _same, config, errors, street

pytestmark = pytest.mark.gpu

GAP = (5, 6, 7)                                   # scans dropped from the second pass: the guess after them is 1.5 m short
JUMP_AT, JUMP_SHIFT, JUMP_TURN = 6, (8.0, -1.5, 0.0), math.radians(40.0)    # a restart 4.7 m ahead, 1.9 m aside, turned 40 degrees
N_UNEXPLAINED = 3


@pytest.fixture(scope="module")
def nl():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    sys.path.insert(0, ROOT)
    import nerfloam_b200
    return nerfloam_b200


def second(nl, i, seed=6000):
    return street(nl, i, seed=seed + i, shift=SHIFT, turn=TURN)


def unexplainable(seed):
    """test_gpu_localise.py's scan the map cannot explain: every return 20-30 m away at 70-85 degrees of elevation."""
    rng = np.random.default_rng(seed)
    n = 6000
    el, az, r = np.deg2rad(rng.uniform(70, 85, n)), rng.uniform(-np.pi, np.pi, n), rng.uniform(20, 30, n)
    pts = (np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1) * r[:, None]).astype(np.float32)
    return pts, np.ones(n, np.float32), None


def drives(nl):
    """name -> list of (points, cos, true pose or None)."""
    gap = [second(nl, i) for i in range(14) if i not in GAP]
    jump = [second(nl, i) for i in range(JUMP_AT)] + [street(nl, k, seed=7000 + k, shift=JUMP_SHIFT, turn=TURN + JUMP_TURN)
                                                      for k in range(6)]
    unexpl = [second(nl, i) for i in range(5)] + [unexplainable(10 + k) for k in range(N_UNEXPLAINED)] + [second(nl, i) for i in range(5, 10)]
    healthy = [second(nl, i) for i in range(10)]
    return {"gap": gap, "jump": jump, "unexplained": unexpl, "healthy": healthy}


@pytest.fixture(scope="module")
def run(nl, tmp_path_factory):
    """Every drive localised in one loaded map, recovery on (and off where a test compares), each with its own seeded generator."""
    tmp = tmp_path_factory.mktemp("recovery")
    s = nl.slam.NeRFLOAM(config(), str(tmp / "run"), data_stream=MemoryStream([street(nl, i, seed=2000 + i) for i in range(N_MAP)], True))
    s.run()
    torch.cuda.synchronize()
    path = tmp / "run.map"
    s.save_map(path)
    del s
    saved = nl.slam.load_map(path)
    before = {k: v.clone() for k, v in _buffers(saved.map.map_states["_mapstate"], saved.decoder).items()}
    out = SimpleNamespace(tmp=tmp, path=path, drives=drives(nl), res={}, loc={}, gen={})
    plan = [("gap", False), ("gap", True), ("jump", True), ("unexplained", True), ("healthy", False), ("healthy", True),
            ("healthy_again", False)]
    for name, on in plan:
        scans = out.drives[name.replace("_again", "")]
        g = torch.Generator().manual_seed(11)
        loc = nl.localise.Localiser(saved, MemoryStream(scans, False), generator=g, config={"recovery_specs": {}} if on else None,
                                    out_dir=str(tmp / f"{name}_{on}"))
        res = loc.run()
        torch.cuda.synchronize()
        key = (name, on)
        out.res[key], out.loc[key], out.gen[key] = res, loc, g.get_state()
        truth = [p for _, _, p in scans]
        known = [k for k, p in enumerate(truth) if p is not None]
        dt, dr = errors(res.poses[known], np.stack([truth[k] for k in known]))
        med = [float(np.median(res.loss[max(0, k - 10):k].numpy())) if k else float("nan") for k in range(len(scans))]
        print(f"\n{name} recovery={'on' if on else 'off'}  status={res.status}")
        print("  translation error (m):", np.round(dt.numpy(), 4).tolist())
        print("  rotation error (Frobenius):", np.round(dr.numpy(), 5).tolist())
        print("  loss:", np.round(res.loss.numpy(), 5).tolist())
        print("  loss / median of the previous 10:", np.round(res.loss.numpy() / np.array(med), 3).tolist())
        print("  hit fraction:", np.round(res.hit_fraction.numpy(), 3).tolist())
        print("  summary:", json.dumps(loc.summary(res)))
    torch.cuda.synchronize()
    out.after = _buffers(saved.map.map_states["_mapstate"], saved.decoder)
    out.before = before
    return out


def _errors(run, key, positions):
    scans = run.drives[key[0].replace("_again", "")]
    return errors(run.res[key].poses[positions], np.stack([scans[k][2] for k in positions]))


def test_gap_of_dropped_scans(nl, run):
    """Without recovery a pose after the gap is out of bounds; with it every pose is in bounds and the scan after the gap is
    re-placed."""
    after = list(range(5, len(run.drives["gap"])))
    dt, dr = _errors(run, ("gap", False), after)
    assert run.res[("gap", False)].status is None
    assert float(dt.max()) > MAX_DT or float(dr.max()) > MAX_DR
    res = run.res[("gap", True)]
    dt, dr = _errors(run, ("gap", True), list(range(len(run.drives["gap"]))))
    assert float(dt.max()) < MAX_DT and float(dr.max()) < MAX_DR
    assert res.status[5] in ("local", "global") and "lost" not in res.status
    lines = (run.tmp / "gap_True" / "frame_status.txt").read_text().splitlines()
    assert lines == [f"{i} {s}" for i, s in zip(res.scan_ids.tolist(), res.status)]
    assert not (run.tmp / "gap_False" / "frame_status.txt").exists()


def test_restart_beyond_the_local_lattice(nl, run):
    res = run.res[("jump", True)]
    assert res.status[JUMP_AT] == "global"
    dt, dr = _errors(run, ("jump", True), list(range(len(run.drives["jump"]))))
    assert float(dt.max()) < MAX_DT and float(dr.max()) < MAX_DR
    sm = run.loc[("jump", True)].summary(res)
    assert sm["recovery"]["counts"]["global"] >= 1 and sm["recovery"]["ms"]["global"] > 0


def test_scans_the_map_cannot_explain_are_lost(nl, run):
    res = run.res[("unexplained", True)]
    bad = list(range(5, 5 + N_UNEXPLAINED))
    assert [res.status[k] for k in bad] == ["lost"] * N_UNEXPLAINED
    assert all(math.isnan(float(res.loss[k])) and float(res.hit_fraction[k]) == 0.0 for k in bad)
    good = [k for k in range(len(res.status)) if k not in bad]
    assert all(res.status[k] != "lost" for k in good)
    dt, dr = _errors(run, ("unexplained", True), good)
    assert float(dt.max()) < MAX_DT and float(dr.max()) < MAX_DR
    # the global search ran once for the run of lost scans (global_interval 5 > 3 scans)
    assert len(run.loc[("unexplained", True)].times["recover_global"]) == 1


def test_healthy_drive_untouched(nl, run):
    """Recovery on a drive that never gets lost: every status tracked, no search and no extra draw from the generator (its state
    after the run is the same as without recovery), and the same results as without recovery.  Tracking sums the pose gradient with
    fp32 atomics, so two runs are bit-identical only when the atomics happen to add in the same order: the results are held to the
    spread of two runs without recovery, at most test_gpu_localise.py's 1 cm and 1e-3 between map sources."""
    on, off, again = run.res[("healthy", True)], run.res[("healthy", False)], run.res[("healthy_again", False)]
    assert on.status == ["tracked"] * len(on.status)
    assert not any(k.startswith("recover_") for k in run.loc[("healthy", True)].times)
    assert torch.equal(run.gen[("healthy", True)], run.gen[("healthy", False)])
    bits = {f: torch.equal(getattr(on, f), getattr(off, f)) for f in ("poses", "loss", "hit_fraction")}
    bits_again = {f: torch.equal(getattr(again, f), getattr(off, f)) for f in ("poses", "loss", "hit_fraction")}
    print("bit-identical, on vs off:", bits, " off vs off:", bits_again)
    if all(bits_again.values()):
        assert all(bits.values())
    dt, dr = errors(on.poses, off.poses)
    assert float(dt.max()) < 0.01 and float(dr.max()) < 1e-3
    sm = run.loc[("healthy", True)].summary(on)
    assert sm["recovery"]["counts"] == {"tracked": len(on.status), "local": 0, "global": 0, "lost": 0}
    assert sm["recovery"]["ms"] == {"local": None, "global": None}
    assert "recovery" not in run.loc[("healthy", False)].summary(off)


def test_map_unchanged(nl, run):
    _same(run.after, run.before)


def test_localise_script_recovers(nl, run):
    seq = run.tmp / "seq"
    os.makedirs(seq / "velodyne", exist_ok=True)
    for i, (pts, _, _) in enumerate(run.drives["gap"][:8]):
        np.concatenate([pts, np.zeros((pts.shape[0], 1), np.float32)], 1).astype(np.float32).tofile(str(seq / "velodyne" / f"{i:06d}.bin"))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "localise.py"), str(run.path), "--data", str(seq), "--out",
                          str(run.tmp / "script"), "--recover"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    summary = json.loads(out.stdout.strip().splitlines()[-1])
    print(summary)
    counts = summary["recovery"]["counts"]
    assert summary["scans"] == 8 and sum(counts.values()) == 8 and counts["local"] + counts["global"] >= 1
    status = [line.split() for line in (run.tmp / "script" / "frame_status.txt").read_text().splitlines()]
    assert [int(i) for i, _ in status] == list(range(8)) and status[5][1] in ("local", "global")
    bad = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "localise.py"), str(run.path), "--data", str(seq),
                          "--recovery-specs", '{"global_interval": 0}'], capture_output=True, text=True, timeout=900)
    assert bad.returncode != 0 and "global_interval" in bad.stderr
