#!/usr/bin/env python
"""Composited, masked refined frames in flight, measured at 512^2 -> 1024^2 (bench.py's stage-1 size, the shipped stage-2 size;
synthetic seed-0 weights) with the seeded stand-in mask networks of oracle/stub_nets.py; stage 2 "exact" and "fast" alternated
over `--rounds` rounds (stage 1 exact), medians and runs reported; one JSON line.

    python tools/composite_refine_bench.py [--steps K] [--warmup W] [--rounds R]

The stand-in networks cost almost nothing, so these numbers measure this project's part of a frame: stage 1, the compositing
and stage-2 mask helpers, the three handoff kernels and stage 2.  What the real MODNet and BiSeNet add is not measured.

  refined_fps[depth]    DriverPipeline(refine=, refine_masks=, composite=masks.face_matte(...)) with `depth` frames in flight
                        (2, 3, 4): K device-resident driver frames over one background, each uint8 frame written to the
                        device; frames/s of wall time
  one_frame_ms          one such frame alone (submit, wait), median over K
  chunked_fps           the chunked path without PIL, as video.drive_image_with_video runs it with the same networks: 16
                        captured stage-1 frames, the matte network and video.connect_img_and_bg at batch 16, then the stage-2
                        masks and Stage2Model.forward at batch 16, and ops.image_to_u8; frames/s of wall time
  pipeline_mb[depth]    device memory (torch.cuda.memory_reserved) one pipeline costs, from an empty cache
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
from refine_stream_bench import CHUNK, DEPTHS, OPTS, S2_SIZE, _release, _wall  # noqa: E402


def stream(pipe, frames, bg, u8, n):
    for i in range(n):
        pipe.submit(frames[i % len(frames)], u8_out=u8[i % len(u8):i % len(u8) + 1], bg=bg)
    pipe.drain()


def chunked(w, s2, nets, bg, batch, n):
    """n frames as the chunked path runs them, minus PIL"""
    from emoportraits_b200 import masks, ops, video

    modnet, face_idt, mask_fn = nets
    for i in range(0, n, CHUNK):
        _, img = w.forward(None, batch[:min(CHUNK, n - i)], crop=False, **OPTS)
        x = video.connect_img_and_bg(img, bg, mask_fn(img))
        _, resized = s2.resize(x)
        _, _, ffhq = s2.forward(x, masks.modnet_get_mask(modnet, resized), face_idt.forward(resized)[0])
        ops.image_to_u8(ffhq)


def measure(w, s2, nets, bg, frames, batch, K, W):
    from emoportraits_b200.infer import DriverPipeline

    modnet, face_idt, mask_fn = nets
    out = {"refined_fps": {}, "pipeline_mb": {}}
    u8 = torch.empty((2 * max(DEPTHS), S2_SIZE, S2_SIZE, 3), dtype=torch.uint8, device="cuda")
    sampler = bench.ClockSampler(torch.cuda.current_device())
    for depth in DEPTHS:
        _release()
        m0 = torch.cuda.memory_reserved()
        pipe = DriverPipeline(w.model, w.identity, depth=depth, refine=s2, refine_masks=dict(modnet=modnet, face_idt=face_idt),
                              composite=mask_fn, **OPTS)
        torch.cuda.synchronize()
        out["pipeline_mb"][depth] = (torch.cuda.memory_reserved() - m0) / 2 ** 20
        stream(pipe, frames, bg, u8, W)
        sampler.start()
        out["refined_fps"][depth] = K * 1000.0 / _wall(lambda: stream(pipe, frames, bg, u8, K), 1)
        if depth == DEPTHS[0]:
            it = iter(range(10 ** 9))
            out["one_frame_ms"] = _wall(lambda: stream(pipe, [frames[next(it) % len(frames)]], bg, u8, 1), K)
        out.setdefault("clocks", []).append(sampler.stop())
        del pipe
    _release()
    chunked(w, s2, nets, bg, batch, CHUNK * max(1, W // CHUNK))
    sampler.start()
    n = CHUNK * max(1, K // CHUNK)
    out["chunked_fps"] = n * 1000.0 / _wall(lambda: chunked(w, s2, nets, bg, batch, n), 1)
    out["clocks"].append(sampler.stop())
    _release()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/composite_refine_bench.py measures on the GPU"
    from emoportraits_b200 import masks
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    card = _card()
    cfg = shipped_config(bench.SIZE)
    w = InferenceWrapper("bench", args_path=ROOT / "tests" / "golden" / f"args_{bench.SIZE}.txt",
                         state_dict=synthetic_state_dict(cfg, 0), head_pose_state_dict=synthetic_head_pose_state_dict(0),
                         print_params=False)
    cfg2 = Stage2Config(output_size=S2_SIZE)
    sd2 = synthetic_state_dict_s2(cfg2, 0)
    s2s = {m: Stage2Model(cfg2, sd2, "cuda", precision=m) for m in ("exact", "fast")}
    face_idt = masks.FaceParsing(None, device="cuda", net=StubBiSeNet().cuda())
    modnet = StubMODNet().cuda()
    nets = (modnet, face_idt, masks.face_matte(masks.FaceParsing(None, device="cuda", net=StubBiSeNet().cuda()), StubMODNet().cuda()))
    w.forward(bench.frame(bench.SIZE, 0).cuda(), None, crop=False)
    frames = [bench.frame(bench.SIZE, 1000 + i).cuda() for i in range(8)]
    bg = bench.frame(bench.SIZE, 7)[0].cuda().contiguous()
    batch = torch.cat([frames[i % len(frames)] for i in range(CHUNK)])
    K, W = args.steps, max(args.warmup, 2)
    runs = {m: [] for m in s2s}
    for _ in range(args.rounds):
        for m, s2 in s2s.items():
            runs[m].append(measure(w, s2, nets, bg, frames, batch, K, W))
    res = {}
    for m, rs in runs.items():
        res[m] = {"refined_fps": {d: statistics.median(r["refined_fps"][d] for r in rs) for d in DEPTHS},
                  "one_frame_ms": statistics.median(r["one_frame_ms"] for r in rs),
                  "chunked_fps": statistics.median(r["chunked_fps"] for r in rs),
                  "pipeline_mb": {d: statistics.median(r["pipeline_mb"][d] for r in rs) for d in DEPTHS},
                  "runs": [{k: r[k] for k in ("refined_fps", "one_frame_ms", "chunked_fps", "pipeline_mb")} for r in rs],
                  "clocks": [r["clocks"] for r in rs]}
    line = {"metric": f"composited, masked refined frames {bench.SIZE}^2 -> {S2_SIZE}^2 (stand-in mask networks): frames/s with "
                      "2 / 3 / 4 in flight, one frame alone, the chunked path (stage 2 at batch 16), memory per pipeline",
            **card, "steps": K, "warmup": W, "rounds": args.rounds, "exact": res["exact"], "fast": res["fast"]}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
