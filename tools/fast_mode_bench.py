#!/usr/bin/env python
"""Exact vs fast mode (decoder on one fp16 operand plane, ops.H1) in the same run on the same card; one JSON line.

    python tools/fast_mode_bench.py [--steps K] [--warmup W] [--rounds R]
    python tools/fast_mode_bench.py --stage2 [--steps K] [--warmup W] [--rounds R]     (stage 2: see main_stage2)
    python tools/fast_mode_bench.py --source [--steps K] [--warmup W] [--rounds R]     (the source pass: see main_source)

Per mode, with bench.py's definitions (driver frame @512^2, shipped model, synthetic seed-0 weights, cached source identity):
  fps          device-resident driver frames/s, four captured frames in flight (infer.DriverPipeline depth 4), CUDA events
  e2e          frames/s with a pinned host frame in and the host image out every step (two frames of host run-ahead per stream)
  latency_ms   one captured frame at a time (depth 1), CUDA events / K
  decoder_conv_ms_graph  the decoder's convolutions per frame: every conv shape of one decoder pass as CUDA-graph replays of 10
               back-to-back launches (mean of the no-residual / residual forms, as bench.py times the frame's convs), weighted
               by its launches per frame
  decoder_ms_graph       one whole decoder pass, CUDA-graph replays
The modes alternate for `--rounds` rounds so that a drift of the card's clocks hits both; the median of the rounds is
reported, with the spread.  The SM clocks during the timed regions are recorded as bench.py records them."""
from __future__ import annotations

import argparse
import json
import math
import pathlib
import re
import statistics
import subprocess
import sys
import time

import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402  (frame(), ClockSampler, SIZE: the benchmark's own definitions)


def graph_time_conv(shape_key: str, reps: int = 10):
    """bench.graph_time_conv for every operand mode of the profiler's shape keys (p2 / p3 / ph2 / ph1)"""
    from emoportraits_b200 import ops

    m = re.match(r"(\d+)x(\d+)x(\d+)x(\d+)x(\d+)->(\d+) k(\d)(\d)(\d) s(\d) p(\w+)( up2-subpixel)?", shape_key)
    N, D, H, W, Ci, Co, kd, kh, kw, st_ = map(int, m.groups()[:10])
    pl, up = m.group(11), m.group(12)
    planes = {"h2": ops.H2, "h1": ops.H1}.get(pl) or int(pl)
    x = torch.randn((N, D, H, W, Ci), device="cuda")
    w = torch.randn((Co, Ci, kd, kh, kw) if kd > 1 else (Co, Ci, kh, kw)) / math.sqrt(Ci * kd * kh * kw)
    a = ops.split_bf16(x, planes)
    pw = ops.pack_upconv_weight(w, planes=planes) if up else ops.pack_conv_weight(w, planes=planes)
    pad = (kd // 2, 1, 1) if kh == 4 else None
    Ho, Wo = (2 * H, 2 * W) if up else ((H + 2 * (1 if kh == 4 else kh // 2) - kh) // st_ + 1, (W + 2 * (1 if kw == 4 else kw // 2) - kw) // st_ + 1)
    out = torch.empty((N, D, Ho, Wo, Co), device="cuda")
    bias = torch.zeros(Co, device="cuda")
    res_full = torch.randn(out.shape, device="cuda") if Co % 4 == 0 else None
    times = []
    for res in (None, res_full):
        ops.begin_pass("cuda")
        stt = ops.new_stats(N, 32, "cuda") if Co % 32 == 0 else None
        run = lambda: ops.conv_igemm(a, pw, stride=(1, st_, st_), pad=pad, out=out, bias=bias, residual=res, stats=stt, upconv=bool(up))
        times.append(_graph_us(run, reps))
    return sum(times) / len(times)


def _graph_us(run, reps, replays=5):
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            run()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (replays * reps) * 1000.0


def decoder_times(model):
    """(graph-timed decoder conv ms per frame, graph-timed whole decoder ms, per-shape table)"""
    from emoportraits_b200 import ops

    cfg, dec = model.cfg, model.decoder_nw
    feat = ops.split_bf16(torch.rand((1, 1, cfg.S, cfg.S, cfg.D * cfg.C), device="cuda"), dec.planes)
    prof = ops.ConvProfiler()
    ops.set_conv_profiler(prof)
    ops.begin_pass("cuda")
    dec(feat)
    torch.cuda.synchronize()
    ops.set_conv_profiler(None)
    table, conv_us = [], 0.0
    for name, n, _ms, _alg, _mma in prof.table():
        us = graph_time_conv(name)
        conv_us += us * n
        table.append({"shape": name, "launches": n, "us_per_launch": us})

    def whole():
        ops.begin_pass("cuda")
        dec(feat)
    dec_us = _graph_us(whole, 1, replays=20)
    return conv_us / 1000.0, dec_us / 1000.0, table


def measure(model, st, frames_host, frames_dev, K, W):
    from emoportraits_b200.infer import DriverPipeline

    out = {}
    pipe = DriverPipeline(model, st, depth=4, mix=True)
    for i in range(W):
        pipe.submit(frames_dev[i % len(frames_dev)])
    pipe.drain()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(K):
        pipe.submit(frames_dev[i % len(frames_dev)])
    pipe.drain()
    e1.record()
    torch.cuda.synchronize()
    out["fps"] = K / (e0.elapsed_time(e1) / 1000.0)
    out["clocks"] = sampler.stop()
    ring = 8
    hosts = [torch.empty((1, 3, bench.SIZE, bench.SIZE)).pin_memory() for _ in range(ring)]
    tickets = [None] * ring

    def step_e2e(i):
        t = tickets[i % ring]
        if t is not None:
            t.done.synchronize()
        tickets[i % ring] = pipe.submit(frames_host[i % len(frames_host)], host_out=hosts[i % ring])

    for i in range(2 * ring):
        step_e2e(i)
    pipe.drain()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(K):
        step_e2e(i)
    pipe.drain()
    torch.cuda.synchronize()
    out["e2e"] = K / (time.perf_counter() - t0)
    del pipe
    lat = DriverPipeline(model, st, depth=1, mix=True)
    for i in range(3):
        lat.submit(frames_dev[i % len(frames_dev)])
    lat.drain()
    torch.cuda.synchronize()
    e0.record()
    for i in range(K):
        lat.submit(frames_dev[i % len(frames_dev)])
    lat.drain()
    e1.record()
    torch.cuda.synchronize()
    out["latency_ms"] = e0.elapsed_time(e1) / K
    return out


def _card():
    props = torch.cuda.get_device_properties(0)
    out = {"gpu": props.name, "sm_count": props.multi_processor_count}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = None
    return out


def stage2_images_per_s(model, img, K, W):
    for _ in range(W):
        model.forward(img)
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        model.forward(img)
    e1.record()
    torch.cuda.synchronize()
    return img.shape[0] * K / (e0.elapsed_time(e1) / 1000.0), sampler.stop()


def stage2_times(model, img):
    """(graph-timed stage-2 convolutions ms per image, per-shape table, stem ms per image: conv_direct, stem_pack + conv_igemm)"""
    from emoportraits_b200 import ops

    B, S = img.shape[0], model.cfg.output_size
    prof = ops.ConvProfiler()
    ops.set_conv_profiler(prof)
    model.forward(img)
    torch.cuda.synchronize()
    ops.set_conv_profiler(None)
    table, conv_us = [], 0.0
    for name, n, _ms, _alg, _mma in prof.table():
        us = graph_time_conv(name)
        conv_us += us * n
        table.append({"shape": name, "launches": n, "us_per_launch": us})
    x4 = ops.resize_bilinear(img, (S, S))
    stem_h1 = ops.pack_stem_weight(model.stem_w.cpu(), device="cuda")
    direct_us = _graph_us(lambda: ops.conv_direct(x4, model.stem_w, 1, 3, model.stem_b), 1, replays=20)
    igemm_us = _graph_us(lambda: ops.conv_igemm(ops.stem_pack(x4), stem_h1, pad=(0, 3, 0), bias=model.stem_b), 1, replays=20)
    return conv_us / 1000.0 / B, table, {"conv_direct": direct_us / 1000.0 / B, "stem_pack+conv_igemm": igemm_us / 1000.0 / B}


def main_stage2(args):
    """Stage 2 exact vs fast with bench.py's stage-2 definition (@1024^2, batch 4, synthetic seed-0 weights, torch.rand 512^2
    input): images/s alternated over the rounds, the stage-2 convolutions graph-timed per image (the ConvProfiler's shapes of
    one forward, each as CUDA-graph replays without its post-op, as decoder_times does), and the 7x7 stem per image both ways."""
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2

    cfg = Stage2Config(output_size=1024)
    sd = synthetic_state_dict_s2(cfg, 0)
    models = {m: Stage2Model(cfg, sd, "cuda", precision=m) for m in ("exact", "fast")}
    torch.manual_seed(0)
    img = torch.rand(4, 3, 512, 512, device="cuda")
    K, W = args.steps, max(args.warmup, 3)
    runs = {m: [] for m in models}
    for _ in range(args.rounds):
        for m in models:
            runs[m].append(stage2_images_per_s(models[m], img, K, W))
    res = {}
    for m, rs in runs.items():
        conv_ms, table, stem = stage2_times(models[m], img)
        res[m] = {"images_per_s": statistics.median(r[0] for r in rs), "images_per_s_runs": [r[0] for r in rs],
                  "conv_ms_per_image_graph": conv_ms, "conv_shapes": table, "clocks": [r[1] for r in rs]}
        if m == "exact":
            res["stem_ms_per_image_graph"] = stem
    with torch.no_grad():
        ffhq = {m: models[m].forward(img)[2] for m in models}
    d = (ffhq["fast"] - ffhq["exact"]).abs()
    u8 = {m: (ffhq[m] * 255).to(torch.uint8) for m in ffhq}
    line = {"metric": "stage-2 fast mode (every convolution on one fp16 operand plane, stem on the tensor cores) vs exact, "
                      "images/s @1024^2 batch 4",
            **_card(), "steps": K, "warmup": W, "rounds": args.rounds, "exact": res["exact"], "fast": res["fast"],
            "speedup": res["fast"]["images_per_s"] / res["exact"]["images_per_s"],
            "conv_speedup_graph": res["exact"]["conv_ms_per_image_graph"] / res["fast"]["conv_ms_per_image_graph"],
            "stem_ms_per_image_graph": res["stem_ms_per_image_graph"],
            "ffhq_vs_exact": {"max_abs": d.max().item(), "mean_abs": d.mean().item(),
                              "uint8_changed": (u8["fast"] != u8["exact"]).float().mean().item()}}
    print(json.dumps(line))


class _Timed:
    """a network of Model whose calls record a CUDA event before and after (on the current stream)"""

    def __init__(self, net, events):
        self.net, self.events = net, events

    def __call__(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.net(*a, **k)
        e1.record()
        self.events.append((e0, e1))
        return out


def source_pass_times(model, src, reps):
    """per source pass (eager, as the wrapper runs it), ms: total and the split LocalEncoder / VolumeSource + the two warps
    (from the start of VolumeSource to the start of Unet3D) / Unet3D / rest; the median of `reps` passes"""
    ev = {k: [] for k in ("le", "vs", "unet")}
    nets = {"le": "local_encoder_nw", "vs": "volume_source_nw", "unet": "volume_process_nw"}
    orig = {k: getattr(model, n) for k, n in nets.items()}
    for k, n in nets.items():
        setattr(model, n, _Timed(orig[k], ev[k]))
    tot = []
    try:
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model.source_pass(src)
            e1.record()
            tot.append((e0, e1))
        torch.cuda.synchronize()
    finally:
        for k, n in nets.items():
            setattr(model, n, orig[k])
    rows = []
    for i in range(reps):
        t = tot[i][0].elapsed_time(tot[i][1])
        le = ev["le"][i][0].elapsed_time(ev["le"][i][1])
        vs = ev["vs"][i][0].elapsed_time(ev["unet"][i][0])
        un = ev["unet"][i][0].elapsed_time(ev["unet"][i][1])
        rows.append(dict(source_pass_ms=t, local_encoder_ms=le, volume_source_and_warps_ms=vs, unet3d_ms=un, rest_ms=t - le - vs - un))
    return {k: statistics.median(r[k] for r in rows) for k in rows[0]}


def photo_to_photo_ms(wrapper, src, drv, reps):
    """wall time of wrapper.forward(source, driver): one source pass and one driver frame, the PIL image back on the host"""
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wrapper.forward(src, drv, crop=False, mix=True, mix_old=False)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1000.0)
    return statistics.median(out)


def main_source(args):
    """The source pass (notebooks/infer.py:374-507) exact vs source_precision="fast" @512^2 (bench.py's size, shipped model,
    synthetic seed-0 weights, bench.frame(512, 0) as the source), the modes alternated over the rounds: the source pass's
    device time per pass split by network (CUDA events, median of --steps passes after --warmup), and photo-to-photo latency,
    InferenceWrapper.forward(source, driver) wall time including the PIL conversion (median of --steps // 4 calls)."""
    import numpy as np

    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper

    cfg = shipped_config(bench.SIZE)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    wrappers = {m: InferenceWrapper("bench", args_path=ROOT / "tests" / "golden" / f"args_{bench.SIZE}.txt", state_dict=sd,
                                    head_pose_state_dict=hsd, print_params=False, source_precision=m) for m in ("exact", "fast")}
    src = bench.frame(bench.SIZE, 0).cuda()
    drv = bench.frame(bench.SIZE, 1000).cuda()
    K, W = args.steps, max(args.warmup, 3)
    runs = {m: [] for m in wrappers}
    for _ in range(args.rounds):
        for m, w in wrappers.items():
            source_pass_times(w.model, src, W)
            photo_to_photo_ms(w, src, drv, 2)
            sampler = bench.ClockSampler(torch.cuda.current_device())
            sampler.start()
            r = source_pass_times(w.model, src, K)
            r["photo_to_photo_ms"] = photo_to_photo_ms(w, src, drv, max(K // 4, 3))
            r["clocks"] = sampler.stop()
            runs[m].append(r)
    res = {}
    keys = ("source_pass_ms", "local_encoder_ms", "volume_source_and_warps_ms", "unet3d_ms", "rest_ms", "photo_to_photo_ms")
    for m, rs in runs.items():
        res[m] = {k: statistics.median(r[k] for r in rs) for k in keys}
        res[m].update(source_pass_ms_runs=[r["source_pass_ms"] for r in rs], photo_to_photo_ms_runs=[r["photo_to_photo_ms"] for r in rs],
                      clocks=[r["clocks"] for r in rs])
    pil, img = {}, {}
    for m, w in wrappers.items():
        pil[m], img[m] = w.forward(src, drv, crop=False, mix=True, mix_old=False)
    d = (img["fast"] - img["exact"]).abs()
    u8 = {m: torch.from_numpy(np.asarray(pil[m][0])).int() for m in pil}
    line = {"metric": "source pass with source_precision=fast (local encoder, volume blocks, 3-D U-Net on one fp16 operand "
                      "plane; stem on the tensor cores) vs exact @512^2: source pass ms, photo-to-photo ms",
            **_card(), "steps": K, "warmup": W, "rounds": args.rounds, "exact": res["exact"], "fast": res["fast"],
            "speedup": {k: res["exact"][k] / res["fast"][k] for k in keys},
            "image_vs_exact": {"max_abs": d.max().item(), "mean_abs": d.mean().item(),
                               "uint8_moved": (u8["fast"] != u8["exact"]).float().mean().item(),
                               "uint8_max_levels": (u8["fast"] - u8["exact"]).abs().max().item()}}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stage2", action="store_true", help="the stage-2 arm (main_stage2) instead of the stage-1 decoder's")
    ap.add_argument("--source", action="store_true", help="the source-pass arm (main_source): source_precision exact vs fast")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/fast_mode_bench.py measures on the GPU"
    if args.stage2:
        main_stage2(args)
        return
    if args.source:
        main_source(args)
        return
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    cfg = shipped_config(bench.SIZE)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    models = {m: Model(cfg, sd, hsd, "cuda", precision=m) for m in ("exact", "fast")}
    src = bench.frame(bench.SIZE, 0).cuda()
    states = {m: models[m].source_pass(src) for m in models}
    frames_host = [bench.frame(bench.SIZE, 1000 + i).pin_memory() for i in range(8)]
    frames_dev = [f.cuda() for f in frames_host]
    K, W = args.steps, max(args.warmup, 3)
    runs = {m: [] for m in models}
    for _ in range(args.rounds):
        for m in models:
            runs[m].append(measure(models[m], states[m], frames_host, frames_dev, K, W))
    res = {}
    for m, rs in runs.items():
        conv_ms, dec_ms, table = decoder_times(models[m])
        res[m] = {k: statistics.median(r[k] for r in rs) for k in ("fps", "e2e", "latency_ms")}
        res[m].update({f"{k}_runs": [r[k] for r in rs] for k in ("fps", "e2e", "latency_ms")})
        res[m].update(decoder_conv_ms_graph=conv_ms, decoder_ms_graph=dec_ms, decoder_conv_shapes=table,
                      clocks=[r["clocks"] for r in rs])
    # the same driver frame through both modes: how far fast mode moves the image
    with torch.no_grad():
        img = {m: models[m].driver_pass(states[m], frames_dev[0], mix=True)[0] for m in models}
    d = (img["fast"] - img["exact"]).abs()
    props = torch.cuda.get_device_properties(0)
    line = {
        "metric": "fast mode (decoder on one fp16 operand plane) vs exact, driver frames @512^2",
        "gpu": props.name, "sm_count": props.multi_processor_count, "steps": K, "warmup": W, "rounds": args.rounds,
        "exact": res["exact"], "fast": res["fast"],
        "speedup": {k: (res["fast"][k] / res["exact"][k]) if k != "latency_ms" else res["exact"][k] / res["fast"][k]
                    for k in ("fps", "e2e", "latency_ms")},
        "decoder_conv_speedup_graph": res["exact"]["decoder_conv_ms_graph"] / res["fast"]["decoder_conv_ms_graph"],
        "image_vs_exact": {"max_abs": d.max().item(), "mean_abs": d.mean().item()},
    }
    try:
        line["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        line["power_limit"] = None
    print(json.dumps(line))


if __name__ == "__main__":
    main()
