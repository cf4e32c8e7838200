#!/usr/bin/env python
"""Driving frames from pose and expression embeddings, measured @512^2 (bench.py's size, shipped model, synthetic seed-0
weights); precision "exact" and "fast" alternated over `--rounds` rounds, medians and runs reported; one JSON line.

    python tools/embedding_drive_bench.py [--steps K] [--warmup W] [--rounds R]

  pose_embed_forward_eager_ms     one call per frame of forward(None, frame, custome_target_pose_embed=e) as it ran before it
                                  was captured: the eager Model.driver_pass, then the uint8 image back on the host
  pose_embed_forward_captured_ms  the same calls through InferenceWrapper.forward (a captured frame); wall time per call
  animate_fps                     InferenceWrapper.animate over K (pose, embedding) pairs, four frames in flight, PIL images
                                  back on the host; frames/s of wall time
  encode_fps                      InferenceWrapper.encode of a device-resident batch of K frames, four in flight; frames/s
  pipeline_mb / capture_ms        device memory (torch.cuda.memory_reserved) and wall time one captured four-slot pipeline
                                  costs, per kind: plain frames, encode, animate, forward with an embedding
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

OPTS = dict(mix=True, mix_old=False)   # the video loop's pose options


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


def eager_forward(w, drv, e):
    """forward(None, drv, custome_target_pose_embed=e) of the parent: the eager pass and the image back on the host"""
    from PIL import Image

    from emoportraits_b200 import ops

    img = w.model.driver_pass(w.identity, w._prep(drv), custom_pose_embed=e, **OPTS)[0]
    return [Image.fromarray(h) for h in ops.image_to_u8(img.contiguous()).cpu().numpy()]


def pipeline_costs(w, frames, theta, pe):
    """memory and capture time of each kind of captured pipeline, from an empty cache"""
    kinds = {"plain": lambda: w.forward(None, frames[0], crop=False, **OPTS),
             "encode": lambda: w.encode(frames[0], **OPTS),
             "animate": lambda: w.animate(tuple(t[:1] for t in theta), pe[:1], **OPTS),
             "pose_embed_forward": lambda: w.forward(None, frames[0], crop=False, custome_target_pose_embed=pe[0], **OPTS)}
    w._pipelines.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    out = {}
    for k, fn in kinds.items():
        m0 = torch.cuda.memory_reserved()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        first = (time.perf_counter() - t0) * 1000.0
        cached = _wall(fn, 3)
        out[k] = {"pipeline_mb": (torch.cuda.memory_reserved() - m0) / 2 ** 20, "capture_ms": first - cached}
    return out


def measure(w, frames, theta, pe, K, W):
    out = {}
    e = pe[0:1]
    n = len(frames)
    for i in range(W):
        eager_forward(w, frames[i % n], e)
        w.forward(None, frames[i % n], crop=False, custome_target_pose_embed=e, **OPTS)
    w.animate(theta, pe, **OPTS)
    w.encode(torch.cat(frames), **OPTS)
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    it = iter(range(10 ** 9))
    out["pose_embed_forward_eager_ms"] = _wall(lambda: eager_forward(w, frames[next(it) % n], e), K)
    out["pose_embed_forward_captured_ms"] = _wall(
        lambda: w.forward(None, frames[next(it) % n], crop=False, custome_target_pose_embed=e, **OPTS), K)
    out["animate_fps"] = K * 1000.0 / _wall(lambda: w.animate(theta, pe, **OPTS), 3)
    batch = torch.cat([frames[i % n] for i in range(K)])
    out["encode_fps"] = K * 1000.0 / _wall(lambda: w.encode(batch, **OPTS), 3)
    out["clocks"] = sampler.stop()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/embedding_drive_bench.py measures on the GPU"
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
    K, W = args.steps, max(args.warmup, 3)
    emb = {}
    for m, w in wrappers.items():
        w.forward(source, None, crop=False)
        theta, pe = w.encode(torch.cat([frames[i % len(frames)] for i in range(K)]), **OPTS)
        emb[m] = (theta, pe)
    costs = {m: pipeline_costs(w, frames, *emb[m]) for m, w in wrappers.items()}
    runs = {m: [] for m in wrappers}
    for _ in range(args.rounds):
        for m, w in wrappers.items():
            runs[m].append(measure(w, frames, *emb[m], K, W))
    res = {}
    scalars = ("pose_embed_forward_eager_ms", "pose_embed_forward_captured_ms", "animate_fps", "encode_fps")
    for m, rs in runs.items():
        res[m] = {k: statistics.median(r[k] for r in rs) for k in scalars}
        res[m]["pipelines"] = costs[m]
        res[m]["runs"] = [{k: r[k] for k in scalars} for r in rs]
        res[m]["clocks"] = [r["clocks"] for r in rs]
    line = {"metric": "driving from embeddings @512^2: forward with custome_target_pose_embed eager vs captured ms per call, "
                      "animate and encode frames/s (four in flight), memory and capture time per captured pipeline",
            **card, "steps": K, "warmup": W, "rounds": args.rounds, "exact": res["exact"], "fast": res["fast"],
            "pose_embed_forward_speedup": {m: res[m]["pose_embed_forward_eager_ms"] / res[m]["pose_embed_forward_captured_ms"]
                                           for m in res}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
