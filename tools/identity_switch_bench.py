#!/usr/bin/env python
"""Switching identities without re-capturing the driver graphs, measured @512^2 (bench.py's size, shipped model, synthetic
seed-0 weights); exact and source_precision="fast" alternated over `--rounds` rounds, medians and runs reported; one JSON line.

    python tools/identity_switch_bench.py [--steps K] [--warmup W] [--rounds R]

  photo_to_photo_ms           InferenceWrapper.forward(source, driver) wall time, PIL image back on the host, with a different
                              source image every call (fast_mode_bench.photo_to_photo_ms otherwise): one source pass, the
                              identity loaded into the kept graphs, one frame
  photo_to_photo_recapture_ms the same calls with the wrapper's pipeline dropped before each one: a fresh DriverPipeline per
                              identity (four captures per call), the behaviour before the graphs loaded identities
  switch_copy_ms              one identity load (replay.load: the identity fields copied into a graph's buffers), CUDA events
                              around K loads alternating between two identities on one stream
  latency_ms / latency_switch_ms  one captured frame at a time (depth 1), CUDA events / K: one identity / a new identity
                              every frame (so each frame includes one load)
  fps                         device-resident frames/s, four captured frames in flight (DriverPipeline depth 4), for n = 1, 2,
                              4 and 8 identities: "round_robin" gives frame i identity i % n (with 2 and 4 identities every
                              slot then keeps one identity), "every_frame_switches" gives it (i + i // 4) % n, so that every
                              slot loads a new identity for every frame (the worst case)
The card's name, power limit and maximum SM clock, and the SM clocks sampled during the timed regions, are reported."""
from __future__ import annotations

import argparse
import json
import pathlib
import statistics
import sys
import time

import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import bench  # noqa: E402  (frame(), ClockSampler, SIZE: the benchmark's own definitions)
from fast_mode_bench import _card  # noqa: E402

DEPTH = 4
N_IDS = (1, 2, 4, 8)


def photo_to_photo_ms(wrapper, sources, drv, reps, recapture=False):
    """median wall time of wrapper.forward(sources[i % n], drv); recapture: the wrapper's captured pipelines are dropped first"""
    out = []
    for i in range(reps):
        if recapture:
            wrapper._pipelines.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wrapper.forward(sources[i % len(sources)], drv, crop=False, mix=True, mix_old=False)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1000.0)
    return statistics.median(out)


def _events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def switch_copy_ms(run, states, K):
    for i in range(4):
        run.load(states[i % 2])
    torch.cuda.synchronize()
    e0, e1 = _events()
    e0.record()
    for i in range(K):
        run.load(states[i % 2])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / K


def pipeline_ms(pipe, frames, ids, K, W):
    """ms per frame over K frames, frame i animating ids(i)"""
    for i in range(W):
        pipe.submit(frames[i % len(frames)], st=ids(i))
    pipe.drain()
    torch.cuda.synchronize()
    e0, e1 = _events()
    e0.record()
    for i in range(K):
        pipe.submit(frames[i % len(frames)], st=ids(i))
    pipe.drain()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / K


def measure(w, sources, states, frames, K, W):
    from emoportraits_b200.infer import DriverPipeline

    model, out = w.model, {}
    drv = frames[0]
    photo_to_photo_ms(w, sources, drv, W)
    photo_to_photo_ms(w, sources, drv, 2, recapture=True)
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    out["photo_to_photo_ms"] = photo_to_photo_ms(w, sources, drv, max(K // 4, 3))
    out["photo_to_photo_recapture_ms"] = photo_to_photo_ms(w, sources, drv, max(K // 20, 3), recapture=True)
    lat = DriverPipeline(model, states[0], depth=1, mix=True)
    out["switch_copy_ms"] = switch_copy_ms(lat.slots[0].run, states, K)
    out["latency_ms"] = pipeline_ms(lat, frames, lambda i: states[0], K, W)
    out["latency_switch_ms"] = pipeline_ms(lat, frames, lambda i: states[i % 2], K, W)
    del lat
    pipe = DriverPipeline(model, states[0], depth=DEPTH, mix=True)
    fps = {}
    for n in N_IDS:
        rr = pipeline_ms(pipe, frames, lambda i: states[i % n], K, W)
        fps[f"{n}_round_robin"] = 1000.0 / rr
        if n > 1:
            fps[f"{n}_every_frame_switches"] = 1000.0 / pipeline_ms(pipe, frames, lambda i: states[(i + i // DEPTH) % n], K, W)
    out["fps"] = fps
    out["clocks"] = sampler.stop()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/identity_switch_bench.py measures on the GPU"
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper

    cfg = shipped_config(bench.SIZE)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    wrappers = {m: InferenceWrapper("bench", args_path=ROOT / "tests" / "golden" / f"args_{bench.SIZE}.txt", state_dict=sd,
                                    head_pose_state_dict=hsd, print_params=False, source_precision=m) for m in ("exact", "fast")}
    sources = [bench.frame(bench.SIZE, i).cuda() for i in range(max(N_IDS))]
    frames = [bench.frame(bench.SIZE, 1000 + i).cuda() for i in range(8)]
    states = {m: [w.model.source_pass(s) for s in sources] for m, w in wrappers.items()}
    K, W = args.steps, max(args.warmup, 3)
    runs = {m: [] for m in wrappers}
    for _ in range(args.rounds):
        for m, w in wrappers.items():
            runs[m].append(measure(w, sources, states[m], frames, K, W))
    res = {}
    scalars = ("photo_to_photo_ms", "photo_to_photo_recapture_ms", "switch_copy_ms", "latency_ms", "latency_switch_ms")
    for m, rs in runs.items():
        res[m] = {k: statistics.median(r[k] for r in rs) for k in scalars}
        res[m]["fps"] = {k: statistics.median(r["fps"][k] for r in rs) for k in rs[0]["fps"]}
        res[m]["runs"] = [{k: r[k] for k in scalars + ("fps",)} for r in rs]
        res[m]["clocks"] = [r["clocks"] for r in rs]
    line = {"metric": "identity switching @512^2: photo-to-photo ms (identity loaded into the kept graphs vs a fresh pipeline per "
                      "identity), one identity load ms, frames/s with four in flight for 1-8 identities",
            **_card(), "steps": K, "warmup": W, "rounds": args.rounds, "exact": res["exact"], "source_fast": res["fast"],
            "photo_to_photo_speedup": {m: res[m]["photo_to_photo_recapture_ms"] / res[m]["photo_to_photo_ms"] for m in res}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
