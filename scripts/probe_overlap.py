"""GPU probe: where the fused frame's main-stream chain spends its time between kernels, without events inside the chain.

Runs the bench configuration (1242x375 KITTI-shaped stream, 0x60000 blocks, 0x100000 + 0x80000 entries, decay maxWeight 1 /
minAge 200, 230-frame pre-roll so partial decay is live, L2 flushed before every frame) and reads the kernels' own %globaltimer
stamps (b200_set_timing(4), b200_diag_read_spans): per kernel the first CTA's entry after its dependency wait and the last warp's
exit. The partial decay's sweep runs on CTAs of its own inside the raycast's grid and is stamped apart from the ray CTAs;
the raycast launch's span covers both. The commit that CTA 0 of k_decay_commit runs beside the replay (rank, elect, unlink, counters)
and the ICP-map kernel on the side stream, which runs beside k_decay_commit, are stamped too. Prints, as medians over the
measured frames, each span, the idle time at each of the four boundaries between launches (next entry - previous exit), the
frame's chain from the first entry to the last exit, the frame's tail after the last ray (to the later of the commit's and the
ICP kernel's exits), and per decay pass the flagged blocks whose reset stores k_decay_commit replayed.

Then mode 3 (an event pair around every launch, which serialises the chain) for the same number of frames: the integrate
kernel's stamp span against its event pair, launch by launch — the check that the stamps time the integrate launch as the
events did — and the smallest step of %globaltimer seen in the stamps.

    python scripts/probe_overlap.py [--frames 200] [--json out.json]
"""
import argparse, ctypes as C, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from dynslam_b200 import engine as E, synth
import bench

NAMES = ["k_mark_prepare", "k_serve_list", "k_integrate", "k_raycast", "decay sweep", "k_decay_commit", "commit (CTA 0)",
         "k_icp"]   # b200_diag_read_spans' slots
CHAIN = ["k_mark_prepare", "k_serve_list", "k_integrate", "k_raycast launch", "k_decay_commit"]             # the launches, in order


def read_spans(eng, n):
    buf = (C.c_uint64 * (n * len(NAMES) * 2))()
    got = eng.lib.b200_diag_read_spans(eng.h, buf, n)
    return np.frombuffer(buf, dtype=np.uint64, count=got * len(NAMES) * 2).reshape(got, len(NAMES), 2).astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--preroll", type=int, default=230)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    W, H = synth.KITTI_W, synth.KITTI_H
    n = args.frames
    total = args.preroll + 2 * n + 4
    frames = bench.gen_frames_parallel(6, 0, total, total * 0.8 + 60.0, max(1, min(16, os.cpu_count() or 2)))
    scene = E.Scene(E.SceneParams(), bench.NUM_BLOCKS, bench.NUM_BUCKETS, bench.EXCESS, device="cuda:0")
    eng = E.Engine(scene, (W, H))
    reco = E.SceneReconstructionEngine(eng)
    rs = E.VisualisationEngine(eng, scene).CreateRenderState((W, H))
    reco.ResetScene(scene)
    points = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    normals = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    flush = torch.zeros(256 * 1024 * 1024 // 4, dtype=torch.int32, device=dev)
    view = lambda f: E.View(torch.from_numpy(f[0]).to(dev), torch.from_numpy(f[1]).to(dev), f[2], f[3])
    idx = 0
    for _ in range(args.preroll):
        eng.process_frame_async(rs, view(frames[idx]), points, normals, decay=bench.DECAY); idx += 1
    eng.sync(rs)
    props = torch.cuda.get_device_properties(dev)
    out = {"device": props.name}

    # ---- mode 4: stamps only, the chain as the benchmark runs it ----
    views = [view(frames[idx + i]) for i in range(n)]; idx += n
    torch.cuda.synchronize()
    eng.sync(rs)
    st0 = eng.stats()
    eng.set_timing(4)
    for v in views:
        flush.add_(1)
        eng.process_frame_async(rs, v, points, normals, decay=bench.DECAY)
    eng.sync(rs)
    st1 = eng.stats()
    sp = read_spans(eng, n)
    eng.set_timing(0)
    replay = (st1.decayReplays - st0.decayReplays) / n
    ok = (sp[:, :, 0] > 0).all(axis=1) & (sp[:, :, 1] > 0).all(axis=1)
    sp = sp[ok]
    us = lambda a: float(np.median(a)) / 1000.0
    spans = {NAMES[k]: us(sp[:, k, 1] - sp[:, k, 0]) for k in range(len(NAMES))}
    rc, sw = NAMES.index("k_raycast"), NAMES.index("decay sweep")
    launch = np.stack([np.minimum(sp[:, rc, 0], sp[:, sw, 0]), np.maximum(sp[:, rc, 1], sp[:, sw, 1])], axis=1)
    ch = np.stack([sp[:, 0], sp[:, 1], sp[:, 2], launch, sp[:, NAMES.index("k_decay_commit")]], axis=1)
    chain_spans = {CHAIN[k]: us(ch[:, k, 1] - ch[:, k, 0]) for k in range(len(CHAIN))}
    gaps = {f"{CHAIN[k]} -> {CHAIN[k + 1]}": us(ch[:, k + 1, 0] - ch[:, k, 1]) for k in range(len(CHAIN) - 1)}
    chain = us(ch[:, -1, 1] - ch[:, 0, 0])
    out.update({"frames": int(ok.sum()), "span_us": spans, "launch_span_us": chain_spans, "idle_us": gaps, "chain_us": chain,
                "sum_of_spans_us": sum(chain_spans.values()), "sum_of_idle_us": sum(gaps.values()),
                "sweep_entry_after_raycast_entry_us": us(sp[:, sw, 0] - sp[:, rc, 0]),
                "sweep_exit_before_raycast_exit_us": us(sp[:, rc, 1] - sp[:, sw, 1]),
                "tail_after_last_ray_us": us(np.maximum(sp[:, NAMES.index("k_decay_commit"), 1], sp[:, NAMES.index("k_icp"), 1]) - launch[:, 1]),
                "replays_per_pass": replay})
    print(f"device {props.name}; {int(ok.sum())} frames with every kernel stamped (medians, us)")
    for k, v in spans.items():
        print(f"  span  {k:<20s} {v:7.2f}")
    print(f"  span  {'k_raycast launch':<20s} {chain_spans['k_raycast launch']:7.2f}   (ray CTAs and sweep CTAs)")
    print(f"  sweep exit before the last ray exit {out['sweep_exit_before_raycast_exit_us']:7.2f}")
    for k, v in gaps.items():
        print(f"  idle  {k:<40s} {v:7.2f}   (negative: the next kernel's first CTA passed its wait before the last warp left)")
    print(f"  chain first entry -> last exit {chain:7.2f}; launch spans {sum(chain_spans.values()):.2f} + idle {sum(gaps.values()):.2f}")
    print(f"  tail: last ray exit -> later of the commit's and k_icp's exits {out['tail_after_last_ray_us']:7.2f}")
    print(f"  flagged blocks per decay pass, replayed after the rays: {replay:.1f}")

    # ---- mode 3: the integrate kernel's stamps against an event pair around each launch (no overlap: events in the chain) ----
    views = [view(frames[idx + i]) for i in range(n)]; idx += n
    torch.cuda.synchronize()
    eng.set_timing(3)
    ev_us = []
    for v in views:
        flush.add_(1)
        eng.process_frame_async(rs, v, points, normals, decay=bench.DECAY)
        eng.sync(rs)
        ev_us += [b - a for name, a, b in eng.trace() if name.startswith("k_integrate")]
    sp3 = read_spans(eng, n)
    eng.set_timing(0)
    st_us = (sp3[:, 2, 1] - sp3[:, 2, 0]) / 1000.0
    m = min(len(ev_us), len(st_us))
    d = np.asarray(st_us[:m]) - np.asarray(ev_us[:m])
    stamps = np.unique(np.concatenate([sp[:, :, 0].ravel(), sp[:, :, 1].ravel()]))
    steps = np.diff(stamps)
    res = int(steps[steps > 0].min()) if (steps > 0).any() else 0
    out.update({"integrate_events_us": float(np.median(ev_us[:m])), "integrate_stamps_us": float(np.median(st_us[:m])),
                "stamp_minus_event_us": {"median": float(np.median(d)), "p10": float(np.percentile(d, 10)), "p90": float(np.percentile(d, 90))},
                "globaltimer_step_ns": res})
    print(f"integrate, mode 3, {m} launches: event pair {np.median(ev_us[:m]):.2f} us, stamps {np.median(st_us[:m]):.2f} us; "
          f"stamps - events: median {np.median(d):.2f}, p10 {np.percentile(d, 10):.2f}, p90 {np.percentile(d, 90):.2f} us")
    print(f"smallest %globaltimer step between distinct stamps: {res} ns")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
