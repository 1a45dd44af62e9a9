"""The multi-volume frame through a volume group (b200_group_frame_async, dynslam_b200/volumes.py GroupStreetVolumes) against the
per-engine calls from Python (StreetVolumes), configs[2] of bench.py on one GPU. Prints one JSON line.

Steady arms, per K, built from the same frames (street of seed 6, K followed cars), pre-rolled until the partial decay
(--max_decay_weight=1 --min_decay_age=200) is live, then timed in alternating rounds, each arm for at least --seconds:
  street         StreetVolumes, a stream per engine (forked and joined through b200_engine_wait_engine)
  group          GroupStreetVolumes, a stream per slot
  group_shared   GroupStreetVolumes, every slot on the static engine's stream
Reported per arm: us per frame (n frames ending in a synchronise), host us per frame spent in the enqueue calls, whether the
host's enqueue bounds the loop (enqueue time >= 90 % of the frame time), and byte identity of every volume's state and the
composite with the street arm. The group arms enqueue frames whose b200_group_car arrays were built beforehand (prepare).

Churn arms: a track starts every --churn frames and the oldest one ends, round robin over the K cars. `create` does what a
new InfiniTamDriver costs today: the old engine destroyed (b200_engine_destroy), a new scene, engine and render state created
and the scene reset (b200_reset_scene). `restart` restarts the group's slot on the device (b200_group_track_start). Neither
reaps the old volume. Frame time = the interval between successive frame submissions with at most two frames in flight (the
host waits for frame f-2's completion event before it submits frame f), so a device drain shows up in the frame it happens in;
reported as p50, p99 and the worst frame.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from dynslam_b200 import engine as E, synth, volumes as V  # noqa: E402
from bench_volumes import render_frames, states  # noqa: E402

W, H = synth.KITTI_W, synth.KITTI_H


def card():
    """name, power limit (W), current and maximum SM clock (MHz), read-only"""
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return name, float(q[0]), float(q[1]), float(q[2])
    except Exception:
        return name, None, None, None


def make_arm(kind, k):
    if kind == "street":
        return V.StreetVolumes(k, W, H, False)
    return V.GroupStreetVolumes(k, W, H, kind == "group_shared")


def feed(kind, vol, frames):
    dev = vol.upload(frames)
    return [vol.prepare(fr) for fr in dev] if kind != "street" else dev


def run_frames(vol, feed_, start, n):
    t0 = time.perf_counter()
    for i in range(start, start + n):
        vol.step(feed_[i % len(feed_)])
    t1 = time.perf_counter()
    vol.synchronize()
    return time.perf_counter() - t0, t1 - t0


def same(sa, sb):
    return all(np.array_equal(np.frombuffer(bytes(a[key]), np.uint8), np.frombuffer(bytes(b[key]), np.uint8))
               for a, b in zip(sa, sb) for key in a)


def bench_k(k, frames, args):
    kinds = ("street", "group", "group_shared")
    sub = [(f[0], f[1], f[2], f[3], f[4][:k]) for f in frames]
    arms = {a: make_arm(a, k) for a in kinds}
    feeds = {a: feed(a, v, sub) for a, v in arms.items()}
    for a, v in arms.items():                      # pre-roll: the partial decay is live after it
        run_frames(v, feeds[a], 0, args.preroll)
    pos = args.preroll
    probe = max(run_frames(arms["street"], feeds["street"], pos, 8)[0], 1e-6) / 8
    for a in kinds[1:]:
        run_frames(arms[a], feeds[a], pos, 8)
    pos += 8
    n = max(8, int(args.seconds / 4 / probe))
    spent, enq, done = {a: 0.0 for a in kinds}, {a: 0.0 for a in kinds}, {a: 0 for a in kinds}
    while min(spent.values()) < args.seconds:
        for a in kinds:                            # alternating rounds on the same frames
            wall, host = run_frames(arms[a], feeds[a], pos, n)
            spent[a] += wall
            enq[a] += host
            done[a] += n
        pos += n
    ref = states(arms["street"])
    res = {}
    for a in kinds:
        us, hu = spent[a] / done[a] * 1e6, enq[a] / done[a] * 1e6
        res[a] = {"us_per_frame": round(us, 1), "host_enqueue_us_per_frame": round(hu, 1), "host_bound": hu >= 0.9 * us,
                  "frames": done[a], "seconds": round(spent[a], 3), "same_bytes_as_street": a == "street" or same(ref, states(arms[a]))}
    res["group_over_street"] = round(res["street"]["us_per_frame"] / res["group"]["us_per_frame"], 3)
    for v in arms.values():
        v.close()
    del arms, feeds
    torch.cuda.empty_cache()
    return res


def churn_arm(kind, k, frames, args):
    """per-frame submission intervals (us) of --churn_frames frames, a track start every args.churn frames"""
    vol = V.StreetVolumes(k, W, H, False) if kind == "create" else V.GroupStreetVolumes(k, W, H, False)
    sub = [(f[0], f[1], f[2], f[3], f[4][:k]) for f in frames]
    fd = vol.upload(sub)
    if kind == "restart":
        fd = [vol.prepare(fr) for fr in fd]
    for i in range(args.preroll):
        vol.step(fd[i % len(fd)])
    vol.synchronize()
    evs = [torch.cuda.Event() for _ in range(3)]
    stream = vol.streams[0] if kind == "create" else vol.stream
    times, oldest = [], 0
    t_prev = time.perf_counter()
    for j in range(args.churn_frames):
        i = args.preroll + j
        if j >= 2:
            evs[(j - 2) % 3].synchronize()                # at most two frames in flight
        if j > 0 and j % args.churn == 0:
            c = 1 + oldest
            if kind == "create":
                with torch.cuda.stream(vol.streams[c]):
                    old = vol.engines[c]
                    sc = E.Scene(E.SceneParams(voxelSize=0.035, mu=1.0, maxW=50), V.CAR_BLOCKS, V.NUM_BUCKETS, V.EXCESS, device="cuda:0")
                    old.close()
                    eng = E.Engine(sc, (W, H), stream=vol.streams[c].cuda_stream)
                    E.SceneReconstructionEngine(eng).ResetScene(sc)
                    vol.scenes[c], vol.engines[c] = sc, eng
                    vol.rs[c] = E.VisualisationEngine(eng, sc).CreateRenderState((W, H))
            else:
                vol.track_start(oldest)
            oldest = (oldest + 1) % k
        vol.step(fd[i % len(fd)])
        evs[j % 3].record(stream)
        t = time.perf_counter()
        times.append((t - t_prev) * 1e6)
        t_prev = t
    vol.synchronize()
    vol.close()
    torch.cuda.empty_cache()
    a = np.array(times[1:])
    return {"p50_us": round(float(np.percentile(a, 50)), 1), "p99_us": round(float(np.percentile(a, 99)), 1),
            "worst_us": round(float(a.max()), 1), "frames": int(a.size), "track_starts": args.churn_frames // args.churn}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cars", default="1,3,7")
    ap.add_argument("--preroll", type=int, default=210)
    ap.add_argument("--seconds", type=float, default=1.0, help="least timed time per arm and K")
    ap.add_argument("--distinct", type=int, default=48, help="distinct frames rendered; the sequence cycles through them")
    ap.add_argument("--workers", type=int, default=min(16, os.cpu_count() or 1))
    ap.add_argument("--churn", type=int, default=20, help="frames between track starts in the churn arms")
    ap.add_argument("--churn_frames", type=int, default=400)
    ap.add_argument("--churn_cars", default="3,7")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_volume_group.py measures on a CUDA device; there is none")
    ks = [int(x) for x in args.cars.split(",")]
    cks = [int(x) for x in args.churn_cars.split(",") if x]
    t0 = time.perf_counter()
    frames = render_frames(args.distinct, max(ks + cks), args.workers)
    t_gen = time.perf_counter() - t0
    name, plimit, sm, maxsm = card()
    out = {"bench": "volume_group_one_gpu", "card": name, "power_limit_w": plimit, "sm_clock_mhz": sm, "max_sm_clock_mhz": maxsm,
           "frame": [W, H], "decay": list(V.DECAY), "preroll": args.preroll, "distinct_frames": args.distinct, "render_s": round(t_gen, 1),
           "k": {}, "churn": {}}
    for k in ks:
        out["k"][str(k)] = bench_k(k, frames, args)
    for k in cks:
        out["churn"][str(k)] = {kind: churn_arm(kind, k, frames, args) for kind in ("create", "restart")}
    out["same_bytes"] = all(r[a]["same_bytes_as_street"] for r in out["k"].values() for a in ("group", "group_shared"))
    _, plimit2, sm2, _ = card()
    out["power_limit_w_after"], out["sm_clock_mhz_after"] = plimit2, sm2
    print(json.dumps(out))


if __name__ == "__main__":
    main()
