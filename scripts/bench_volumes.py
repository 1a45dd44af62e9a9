"""The static map and K car volumes on one GPU (dynslam_b200/volumes.py), configs[2] of bench.py on a single device: per-frame
time of (A) every engine on one shared stream, the volumes one after another, against (B) one stream per engine, forked and
joined through b200_engine_wait_engine, the volumes concurrent. Prints one JSON line.

Per K: both arms are built from the same frames (street of seed 6, K followed cars, silhouettes cut on the device), pre-rolled
until the partial decay (--max_decay_weight=1 --min_decay_age=200, DynSLAM's defaults) is live, then timed in alternating
rounds on the same frame sequence, each arm for at least --seconds in all. Afterwards every volume's state (checkpoint, ray
points, raycast image, ICP maps) and the composite are compared between the arms byte for byte (`parity`).

A synthetic frame at KITTI size costs about a second of CPU to render, so --distinct frames are rendered (in parallel) and
the sequence cycles through them; the cycle is the same for both arms.
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dynslam_b200 import synth, volumes as V  # noqa: E402


def _frames(args):
    first, count, ncars = args
    return V.street_frames(first, count, ncars)


def render_frames(count, ncars, workers):
    chunk = (count + workers - 1) // workers
    jobs = [(i * chunk, min(chunk, count - i * chunk), ncars) for i in range(workers) if i * chunk < count]
    with mp.get_context("fork").Pool(len(jobs)) as pool:
        return [f for part in pool.map(_frames, jobs) for f in part]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return name, float(q[0]), float(q[1])
    except Exception:
        return name, None, None


def run_frames(vol, dev_frames, start, n):
    """(wall seconds of n frames ending in a synchronise, host seconds spent enqueueing them). When the enqueue time comes
    close to the wall time, the host's enqueue rate, not the GPU, bounds the loop."""
    t0 = time.perf_counter()
    for i in range(start, start + n):
        vol.step(dev_frames[i % len(dev_frames)])
    t1 = time.perf_counter()
    vol.synchronize()
    return time.perf_counter() - t0, t1 - t0


def states(vol):
    out = [vol.state(i) for i in range(1 + vol.ncars)]
    out.append({"composite colour": vol.out_color.cpu().numpy().tobytes(), "composite depth": vol.out_depth.cpu().numpy().tobytes()})
    return out


def bench_k(k, frames, args):
    arms = {"A": V.StreetVolumes(k, synth.KITTI_W, synth.KITTI_H, True), "B": V.StreetVolumes(k, synth.KITTI_W, synth.KITTI_H, False)}
    dev = {a: v.upload([(f[0], f[1], f[2], f[3], f[4][:k]) for f in frames]) for a, v in arms.items()}
    for a, v in arms.items():                                  # pre-roll: the partial decay is live after it
        run_frames(v, dev[a], 0, args.preroll)
    pos = args.preroll
    # round length from a warm probe of the slower arm, about a quarter of the time per arm
    probe = max(run_frames(arms["A"], dev["A"], pos, 8)[0], 1e-6) / 8
    run_frames(arms["B"], dev["B"], pos, 8)
    pos += 8
    n = max(8, int(args.seconds / 4 / probe))
    spent, enqueue = {"A": 0.0, "B": 0.0}, {"A": 0.0, "B": 0.0}
    frames_done = {"A": 0, "B": 0}
    while min(spent.values()) < args.seconds:
        for a in ("A", "B"):                                   # alternating rounds on the same frames
            wall, host = run_frames(arms[a], dev[a], pos, n)
            spent[a] += wall
            enqueue[a] += host
            frames_done[a] += n
        pos += n
    res = {}
    for a in ("A", "B"):
        us = spent[a] / frames_done[a] * 1e6
        res[a] = {"us_per_frame": round(us, 1), "fps": round(1e6 / us, 2), "frames": frames_done[a], "seconds": round(spent[a], 3),
                  "host_enqueue_us_per_frame": round(enqueue[a] / frames_done[a] * 1e6, 1)}
    res["B_over_A"] = round(res["A"]["us_per_frame"] / res["B"]["us_per_frame"], 3)
    sa, sb = states(arms["A"]), states(arms["B"])
    res["parity"] = all(a[key] == b[key] if not isinstance(a[key], np.ndarray) else np.array_equal(a[key], b[key])
                        for a, b in zip(sa, sb) for key in a)
    for v in arms.values():
        v.close()
    del arms, dev
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cars", default="1,3,7")
    ap.add_argument("--preroll", type=int, default=210)
    ap.add_argument("--seconds", type=float, default=1.0, help="least timed time per arm and K")
    ap.add_argument("--distinct", type=int, default=48, help="distinct frames rendered; the sequence cycles through them")
    ap.add_argument("--workers", type=int, default=min(16, os.cpu_count() or 1))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_volumes.py measures on a CUDA device; there is none")
    ks = [int(x) for x in args.cars.split(",")]
    t0 = time.perf_counter()
    frames = render_frames(args.distinct, max(ks), args.workers)
    t_gen = time.perf_counter() - t0
    name, plimit, maxsm = card()
    out = {"bench": "volumes_one_gpu", "card": name, "power_limit_w": plimit, "max_sm_clock_mhz": maxsm,
           "frame": [synth.KITTI_W, synth.KITTI_H], "decay": list(V.DECAY),
           "preroll": args.preroll, "distinct_frames": args.distinct, "render_s": round(t_gen, 1), "k": {}}
    for k in ks:
        out["k"][str(k)] = bench_k(k, frames, args)
    out["parity"] = all(r["parity"] for r in out["k"].values())
    name2, plimit2, _ = card()
    out["power_limit_w_after"] = plimit2
    print(json.dumps(out))


if __name__ == "__main__":
    main()
