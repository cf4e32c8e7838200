#!/usr/bin/env python
"""Smoothed driver frames (smooth_pose) in flight, measured @512^2 (bench.py's size, shipped model, synthetic seed-0 weights);
precision "exact" and "fast" alternated over `--rounds` rounds, medians and runs reported; one JSON line.

    python tools/smooth_flight_bench.py [--steps K] [--warmup W] [--rounds R]

  forward_single_smoothed_fps  forward(None, frame, smooth_pose=True), one uint8 numpy frame per call: one captured graph
                               per frame, one frame after another (the path of single frames); frames/s of wall time
  forward_list_smoothed_fps    forward(None, [K frames], smooth_pose=True): four frames in flight, each split around its
                               pose step; frames/s of wall time, PIL images back on the host
  forward_list_plain_fps       forward(None, [K frames]) without smoothing: the ceiling of the line above
  pipeline_plain_fps           DriverPipeline(depth=4) over K device-resident frames, CUDA events: the ceiling of the
                               smoothing pipeline
  pipeline_tracks_fps          DriverPipeline(depth=4, smooth=True) over the same frames with n = 1, 2, 4, 8 PoseTracks,
                               frame i on track i mod n
The card's name, power limit and maximum SM clock, and the SM clocks sampled during the timed regions, are reported."""
from __future__ import annotations

import argparse
import json
import pathlib
import statistics
import sys
import time

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import bench  # noqa: E402  (frame(), ClockSampler, SIZE: the benchmark's own definitions)
from fast_mode_bench import _card  # noqa: E402

OPTS = dict(mix=True, mix_old=False)   # the video loop's pose options
DEPTH = 4
N_TRACKS = (1, 2, 4, 8)


def _wall(fn, reps):
    """median wall time (ms) of fn() over reps calls, each ended by a device synchronisation"""
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1000.0)
    return statistics.median(out)


def pipeline_fps(pipe, frames, tracks, K, W):
    """frames/s over K device-resident frames, frame i on tracks(i) (None: a plain pipeline), CUDA events"""
    def run(n):
        for i in range(n):
            tr = tracks(i)
            pipe.submit(frames[i % len(frames)], **({} if tr is None else dict(track=tr)))
        pipe.drain()

    run(W)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(K)
    e1.record()
    torch.cuda.synchronize()
    return K * 1000.0 / e0.elapsed_time(e1)


def measure(w, np_frames, frames, K, W):
    from emoportraits_b200.infer import DriverPipeline

    out = {}
    n = len(np_frames)
    clip = [np_frames[i % n] for i in range(K)]
    it = iter(range(10 ** 9))
    single = lambda: w.forward(None, np_frames[next(it) % n], crop=False, smooth_pose=True, **OPTS)   # noqa: E731
    for _ in range(W):
        single()
    w.forward(None, clip[:2 * DEPTH], crop=False, smooth_pose=True, **OPTS)
    w.forward(None, clip[:2 * DEPTH], crop=False, **OPTS)
    plain = DriverPipeline(w.model, w.identity, depth=DEPTH, **OPTS)
    smooth = DriverPipeline(w.model, w.identity, depth=DEPTH, smooth=True, **OPTS)
    tracks = [smooth.track(momentum=w.pose_momentum) for _ in range(max(N_TRACKS))]
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    out["forward_single_smoothed_fps"] = 1000.0 / _wall(single, K)
    out["forward_list_smoothed_fps"] = K * 1000.0 / _wall(lambda: w.forward(None, clip, crop=False, smooth_pose=True, **OPTS), 3)
    out["forward_list_plain_fps"] = K * 1000.0 / _wall(lambda: w.forward(None, clip, crop=False, **OPTS), 3)
    out["pipeline_plain_fps"] = pipeline_fps(plain, frames, lambda i: None, K, W)
    out["pipeline_tracks_fps"] = {str(t): pipeline_fps(smooth, frames, lambda i, t=t: tracks[i % t], K, W) for t in N_TRACKS}
    out["clocks"] = sampler.stop()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/smooth_flight_bench.py measures on the GPU"
    from emoportraits_b200 import ops
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper

    card = _card()
    cfg = shipped_config(bench.SIZE)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    wrappers = {m: InferenceWrapper("bench", args_path=ROOT / "tests" / "golden" / f"args_{bench.SIZE}.txt", state_dict=sd,
                                    head_pose_state_dict=hsd, print_params=False, precision=m) for m in ("exact", "fast")}
    source = bench.frame(bench.SIZE, 0).cuda()
    frames = [bench.frame(bench.SIZE, 1000 + i).cuda() for i in range(8)]
    np_frames = [np.ascontiguousarray(ops.image_to_u8(f.contiguous()).cpu().numpy()[0]) for f in frames]   # what a camera gives
    K, W = args.steps, max(args.warmup, 2 * DEPTH)
    for w in wrappers.values():
        w.forward(source, None, crop=False)
    runs = {m: [] for m in wrappers}
    for _ in range(args.rounds):
        for m, w in wrappers.items():
            runs[m].append(measure(w, np_frames, frames, K, W))
    res = {}
    scalars = ("forward_single_smoothed_fps", "forward_list_smoothed_fps", "forward_list_plain_fps", "pipeline_plain_fps")
    for m, rs in runs.items():
        res[m] = {k: statistics.median(r[k] for r in rs) for k in scalars}
        res[m]["pipeline_tracks_fps"] = {t: statistics.median(r["pipeline_tracks_fps"][t] for r in rs)
                                         for t in rs[0]["pipeline_tracks_fps"]}
        res[m]["runs"] = [{k: r[k] for k in scalars + ("pipeline_tracks_fps",)} for r in rs]
        res[m]["clocks"] = [r["clocks"] for r in rs]
    line = {"metric": "smoothed driver frames @512^2: forward one frame per call vs a list with four in flight, DriverPipeline "
                      "with 1/2/4/8 pose tracks, plain frames in flight as the ceiling; frames/s",
            **card, "steps": K, "warmup": W, "rounds": args.rounds, "exact": res["exact"], "fast": res["fast"],
            "list_speedup": {m: res[m]["forward_list_smoothed_fps"] / res[m]["forward_single_smoothed_fps"] for m in res}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
