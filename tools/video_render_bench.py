"""End-to-end demo video, two ways, on a seeded synthetic 1080p mp4 (stage 1 at 512^2, stage 2 to 1024^2, composited over a
background, fixed crop box):

  (a) the notebook's way: get_video_frames_as_images + drive_image_with_video(in_flight=True, crop_box=) + make_video
      (decode, resizes, crops and the side-by-side rows in PIL on the host; every refined frame kept as a PIL image);
  (b) video.render_video: the same frames decoded on the host and uploaded, every resize, crop and row on the device.

The arms alternate over --rounds, for stage 2 exact and fast.  Each timing covers the whole video: decoding, the frames, and
writing the mp4.  Reported per arm: wall time, frames/s, peak host RSS (sampled during the arm), peak device memory; and the
card's name, power limit and SM clocks, read in the same run.  A separate untimed pass feeds a few frames of both arms
through a recording writer and checks that their rows are equal.  The mask networks and the inpainter are seeded stand-ins
(oracle/stub_nets.py, tests/test_video_render_gpu.py), so what real networks cost is not measured.

    python tools/video_render_bench.py --rounds 3 [--frames 60] [--out DIR]   (DIR/result.json: the JSON line printed last)
"""
from __future__ import annotations

import argparse
import json
import pathlib
import shutil
import subprocess
import sys
import tempfile
import threading
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

CROP = (128, 64, 896, 960)   # a fixed crop box on the 1024^2 output, as cell 46 computes it from the first frame


def _rss_mb() -> float:
    for line in open("/proc/self/status"):
        if line.startswith("VmRSS:"):
            return int(line.split()[1]) / 1024.0
    return float("nan")


class _PeakRSS:
    """peak resident set size of this process while the block runs, sampled every 5 ms"""

    def __enter__(self):
        self.peak, self.stop = _rss_mb(), False
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()
        return self

    def _run(self):
        while not self.stop:
            self.peak = max(self.peak, _rss_mb())
            time.sleep(0.005)

    def __exit__(self, *a):
        self.stop = True
        self.t.join()


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, sm, sm_max = [s.strip() for s in out[0].split(",")] if out else ("?",) * 4
    return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max, torch_name=torch.cuda.get_device_name())


def _write_mp4(path, n, seed=0):
    """a seeded 1920x1080 mp4: a smooth moving field, so the encoder and the resizes see image-like content"""
    import cv2

    rng = np.random.default_rng(seed)
    base = rng.random((9, 16, 3)).astype(np.float32)
    wr = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), 30.0, (1920, 1080))
    for i in range(n):
        f = cv2.resize(np.roll(base, i % 16, axis=1), (1920, 1080), interpolation=cv2.INTER_CUBIC)
        wr.write(np.clip(f * 255, 0, 255).astype(np.uint8))
    wr.release()


def _setup(root):
    from emoportraits_b200 import masks
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper
    from emoportraits_b200.stage2 import InferenceWrapper as S2Wrapper
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2
    from oracle import frames as FR
    from oracle.stub_nets import StubBiSeNet, StubMODNet
    from test_video_render_gpu import StandInInpainter

    cfg = shipped_config(512)
    w = InferenceWrapper("bench", args_path=ROOT / "tests" / "golden" / "args_512.txt", state_dict=synthetic_state_dict(cfg, 0),
                         head_pose_state_dict=synthetic_head_pose_state_dict(0), print_params=False)
    exp = root / "logs_s2" / "exp"
    (exp / "checkpoints").mkdir(parents=True)
    (exp / "args.txt").write_text((ROOT / "tests" / "golden" / "args_s2_1024.txt").read_text())
    torch.save(synthetic_state_dict_s2(Stage2Config(output_size=1024), 0), exp / "checkpoints" / "m.pth")
    s2 = {p: S2Wrapper(experiment_name="exp", model_file_name="m.pth", project_dir=str(root), precision=p) for p in ("exact", "fast")}
    for s in s2.values():
        s.modnet, s.face_idt = StubMODNet().cuda(), masks.FaceParsing(None, device="cuda", net=StubBiSeNet().cuda())
    mask_fn = masks.face_matte(masks.FaceParsing(None, device="cuda", net=StubBiSeNet().cuda()), StubMODNet().cuda())
    source = FR.pil(512, 41, "smooth")
    from emoportraits_b200 import video

    bg, _ = video.get_bg(source, StandInInpainter().cuda(), mask_fn, 512)
    return w, s2, mask_fn, source, bg


def _arm_a(w, s2w, mask_fn, source, bg, mp4, out):
    from emoportraits_b200 import video

    frames = video.get_video_frames_as_images(mp4, 512)
    _, crops, frames = video.drive_image_with_video(w, source, frames, s2w, bg=bg, mask_fn=mask_fn, crop_box=CROP, in_flight=True)
    video.make_video(source, frames, crops, out, size=512)
    return len(crops)


def _arm_b(w, s2w, mask_fn, source, bg, mp4, out):
    from emoportraits_b200 import video

    w.forward(source, None, crop=False)   # the source pass drive_image_with_video runs itself
    return video.render_video(w, source, mp4, out, s2w, bg=bg, mask_fn=mask_fn, crop_box=CROP, size=512)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--check-frames", type=int, default=6)
    ap.add_argument("--out", default=None, help="also write the result to DIR/result.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("video_render_bench needs a CUDA device")
    import cv2

    tmp = pathlib.Path(tempfile.mkdtemp(prefix="video_render_bench_"))
    try:
        _run(a, tmp, cv2)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def _run(a, tmp, cv2):
    mp4 = tmp / "driver_1080p.mp4"
    _write_mp4(mp4, a.frames)
    short = tmp / "short.mp4"
    _write_mp4(short, a.check_frames, seed=1)
    w, s2, mask_fn, source, bg = _setup(tmp)
    arms = {"a_notebook": _arm_a, "b_render_video": _arm_b}
    res = dict(card=_card(), frames=a.frames, rounds=a.rounds, shape="1920x1080 mp4 -> stage 1 512^2 -> stage 2 1024^2 -> 1536x512 rows",
               runs={})

    # untimed: the rows of both arms through a recording writer
    real_writer = cv2.VideoWriter
    rows = {}

    class Recorder:
        def __init__(self, *args):
            self.rows = rows.setdefault(self.arm, [])

        def write(self, row):
            self.rows.append(np.array(row))

        def release(self):
            pass

    equal = {}
    for prec, s2w in s2.items():
        rows.clear()
        for name, fn in arms.items():
            Recorder.arm = name
            cv2.VideoWriter = Recorder
            try:
                fn(w, s2w, mask_fn, source, bg, str(short), tmp / "x.mp4")
            finally:
                cv2.VideoWriter = real_writer
        ra, rb = rows["a_notebook"], rows["b_render_video"]
        equal[prec] = len(ra) == len(rb) == a.check_frames and all(np.array_equal(x, y) for x, y in zip(ra, rb))
    res["rows_equal"] = equal

    for prec, s2w in s2.items():                                   # warm-up: captures, tables, cuDNN plans
        for name, fn in arms.items():
            fn(w, s2w, mask_fn, source, bg, str(short), tmp / "warm.mp4")
    for r in range(a.rounds):
        for prec, s2w in s2.items():
            for name, fn in arms.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                rss0 = _rss_mb()
                with _PeakRSS() as rss:
                    t0 = time.perf_counter()
                    n = fn(w, s2w, mask_fn, source, bg, str(mp4), tmp / f"{name}_{prec}.mp4")
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                run = res["runs"].setdefault(f"{prec}/{name}", [])
                run.append(dict(seconds=round(dt, 3), frames_per_s=round(n / dt, 2), frames=n, rss_start_mb=round(rss0, 1), peak_rss_mb=round(rss.peak, 1),
                                peak_device_mb=round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)))
                print(prec, name, run[-1], flush=True)
    res["median_frames_per_s"] = {k: float(np.median([x["frames_per_s"] for x in v])) for k, v in res["runs"].items()}
    res["card_after"] = _card()
    if a.out is not None:
        outdir = pathlib.Path(a.out)
        outdir.mkdir(parents=True, exist_ok=True)
        (outdir / "result.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
