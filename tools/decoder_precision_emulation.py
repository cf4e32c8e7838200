"""CPU emulation behind the error budget of the decoder's one-plane fp16 operand mode (ops.H1, DESIGN.md section 2).

    python tools/decoder_precision_emulation.py [size ...] [--frames noise|smooth]     (default: 256 512, noise)
    python tools/decoder_precision_emulation.py --stage2 [size ...] [--frames noise|smooth]
                                                  (stage-2 fast mode; default: 512 1024, smooth and noise; see stage2_main)
    python tools/decoder_precision_emulation.py --source [size ...] [--frames noise|smooth]
                                                  (source-pass fast mode, alone and with the decoder's; default: 256 512,
                                                   smooth and noise; see source_main)

The oracle restatement (oracle/restatement.py, torch fp32 on the CPU) is run to the decoder's input (`aligned_volume`), then
the oracle decoder is run once in exact fp32 and once per operand format with every F.conv2d's input and weights rounded to
that format: bf16 x2 (the default path, three products hi*hi + hi*lo + lo*hi: the calibration row), one fp16 plane of
(value x 16) / (weight x 256) (ops.H1), one bf16 plane.  The products are summed in fp64, so the rows isolate the operand
error (the kernel adds ~1e-6 relative of truncating accumulation).  The emulation also rounds the 128 -> 3 image head, which
the device keeps in exact fp32 (ops.gn_head), so its numbers are slightly pessimistic.

Printed per size and format: image max-abs / mean-abs error, PSNR against the fp32 image, logits max-abs error, and the share
of uint8 output pixels (trunc(clamp(x, 0, 1) * 255), the wrapper's conversion) that change.  tests/test_fast_decoder_gpu.py
takes its decoder bounds from these numbers (synthetic seed-0 weights, oracle frames 21 / 22)."""
import math
import pathlib
import sys

import torch
import torch.nn.functional as F

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

# name -> (plane dtype, planes, products (i, j) of activation plane i and weight plane j, activation scale, weight scale)
FORMATS = {
    "bf16 x2 (3 MMAs, default)": (torch.bfloat16, 2, [(0, 0), (0, 1), (1, 0)], 1.0, 1.0),
    "fp16 x1 scaled (1 MMA, h1)": (torch.float16, 1, [(0, 0)], 16.0, 256.0),
    "bf16 x1 (1 MMA)": (torch.bfloat16, 1, [(0, 0)], 1.0, 1.0),
}


def planes(x, dt, n, scale):
    out, r = [], (x * scale).float()
    for _ in range(n):
        p = r.to(dt)
        out.append(p.double() / scale)
        r = r - p.float()
    return out


def emulated_conv2d(fmt, conv2d):
    dt, n, terms, sa, sw = FORMATS[fmt]

    def wrapped(x, w, b=None, *a, **k):
        xp, wp = planes(x, dt, n, sa), planes(w, dt, n, sw)
        y = sum(conv2d(xp[i], wp[j], None, *a, **k) for i, j in terms)
        if b is not None:
            y = y + b.double().view(1, -1, *([1] * (y.dim() - 2)))
        return y.float()
    return wrapped


def to_u8(img):
    return (img.clamp(0, 1) * 255).to(torch.uint8)


# stage 2 (--stage2): name -> (format of the 7x7 RGB stem, format of every other convolution); None = exact fp32
STAGE2_FORMATS = {
    "bf16 x2, stem fp32 (exact mode)": (None, "bf16 x2 (3 MMAs, default)"),
    "h1, stem fp32": (None, "fp16 x1 scaled (1 MMA, h1)"),
    "h1, stem h1 too (fast mode)": ("fp16 x1 scaled (1 MMA, h1)", "fp16 x1 scaled (1 MMA, h1)"),
}


def forward(R, sd, img, size):
    """R.stage2_forward, also returning the latent: (latent, add, ffhq)"""
    resized = F.interpolate(img, mode="bilinear", size=(size, size), align_corners=False)
    vol = R.stage2_local_encoder(sd, resized)
    add = R.stage2_decoder(sd, vol)
    return vol, add, (resized + add).clamp(min=0, max=1)


def stage2_main(sizes, kinds):
    """Stage-2 fast mode (stage2.Stage2Model(precision="fast")): the oracle stage2_forward, synthetic seed-0 weights, oracle
    frame 21 (512^2) as the input image, with every F.conv2d of the refinement network evaluated in each STAGE2_FORMATS
    row.  The stem's operands are rounded as emo_stem_pack and the packed stem weight round them (fp16(16 x), fp16(256 w)).
    The device folds the pooled 3x3 convolutions into 4x4 stride-2 ones and the up-sampling 3x3 convolutions into sub-pixel
    2x2 ones before it rounds their weights; the emulation rounds the unfolded weights.  Printed against the fp32 result:
    ffhq max-abs / mean-abs, PSNR, uint8 pixels changed (trunc(x * 255), the wrapper's conversion), `add` max-abs, the latent's
    max-abs error and largest magnitude, and the largest |activation| / |weight| any convolution reads."""
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2
    from oracle import frames as FR
    from oracle import restatement as R

    conv2d = F.conv2d
    for size in sizes:
        cfg = Stage2Config(output_size=size)
        sd = synthetic_state_dict_s2(cfg, 0)
        for kind in kinds:
            img = FR.frame(512, 21, kind)
            seen = {"x": 0.0, "w": 0.0}

            def watch(x, w, *a, **k):
                seen["x"] = max(seen["x"], x.abs().max().item())
                seen["w"] = max(seen["w"], w.abs().max().item())
                return conv2d(x, w, *a, **k)

            with torch.no_grad():
                F.conv2d = watch
                try:
                    vol0, add0, ffhq0 = forward(R, sd, img, size)
                finally:
                    F.conv2d = conv2d
                print(f"{size}^2 {kind:6s} largest |activation| into a conv {seen['x']:.2f}, |weight| {seen['w']:.3f}", flush=True)
                for name, (stem_fmt, fmt) in STAGE2_FORMATS.items():
                    body = emulated_conv2d(fmt, conv2d)
                    stem = emulated_conv2d(stem_fmt, conv2d) if stem_fmt else conv2d
                    F.conv2d = lambda x, w, *a, **k: (stem if w.shape[1] == 3 else body)(x, w, *a, **k)
                    try:
                        vol, add, ffhq = forward(R, sd, img, size)
                    finally:
                        F.conv2d = conv2d
                    err = (ffhq - ffhq0).abs()
                    mse = (err ** 2).mean().item()
                    psnr = 10 * math.log10(1.0 / mse) if mse > 0 else float("inf")
                    u8, u80 = (ffhq * 255).to(torch.uint8), (ffhq0 * 255).to(torch.uint8)
                    changed = (u8 != u80).float().mean().item()
                    levels = (u8.int() - u80.int()).abs().max().item()
                    e_vol = (vol - vol0).abs().max().item()
                    print(f"{size}^2 {kind:6s} {name:32s} ffhq max-abs {err.max().item():.1e} mean-abs {err.mean().item():.1e}  "
                          f"PSNR {psnr:5.1f} dB  uint8 pixels changed {100 * changed:.2f} % (at most {levels} level)  "
                          f"add max-abs {(add - add0).abs().max().item():.1e}  latent max-abs {e_vol:.1e} (of max {vol0.abs().max().item():.1f})", flush=True)


# source pass (--source): name -> (format of the local encoder / volume blocks / 3-D U-Net convolutions, of the decoder's)
H1_FMT = "fp16 x1 scaled (1 MMA, h1)"
SOURCE_FORMATS = {
    "source h1 (source_precision=fast)": (H1_FMT, None),
    "decoder h1 (precision=fast)": (None, H1_FMT),
    "source h1 + decoder h1 (both fast)": (H1_FMT, H1_FMT),
}


def source_main(sizes, kinds):
    """Source-pass fast mode (InferenceWrapper(source_precision="fast")): the oracle source pass (synthetic seed-0 weights,
    oracle frame 21) and driver pass (frame 22), with every F.conv2d / F.conv3d of local_encoder, volume_source and unet3d
    evaluated on one fp16 plane, fp16(16 x) and fp16(256 w), products summed in fp64; the 7x7 RGB stem is rounded the same
    way (emo_stem_pack and the packed stem weight round it so).  Everything else runs in exact fp32.  The device folds the
    pooled 3x3 convolutions into 4x4 stride-2 ones before it rounds their weights; the emulation rounds the unfolded weights.
    Rows: the source networks alone, the decoder alone (precision="fast", for comparison) and both together; the decoder's
    128 -> 3 image head stays in fp32, as ops.gn_head keeps it on the device.  Printed against the fp32 result: image max-abs
    / mean-abs, PSNR, uint8 pixels moved (trunc(clamp(x, 0, 1) * 255), the wrapper's conversion) and the largest move,
    `target_latent_volume` max-abs error (of its largest magnitude), and the largest |activation| / |weight| any source
    convolution reads."""
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from oracle import frames as FR
    from oracle import restatement as R

    conv2d, conv3d = F.conv2d, F.conv3d
    nets = {name: getattr(R, name) for name in ("local_encoder", "volume_source", "unet3d", "decoder")}
    where = [None]      # the oracle network being evaluated

    def scoped(name):
        def run(*a, **k):
            where[0] = name
            try:
                return nets[name](*a, **k)
            finally:
                where[0] = None
        return run

    def install(src_fmt, dec_fmt, seen=None):
        def pick(base):
            src = emulated_conv2d(src_fmt, base) if src_fmt else base
            dec = emulated_conv2d(dec_fmt, base) if dec_fmt else base

            def conv(x, w, *a, **k):
                if where[0] == "decoder":
                    return (dec if w.shape[0] > 4 else base)(x, w, *a, **k)     # the image head stays fp32 (ops.gn_head)
                if where[0] is not None:
                    if seen is not None:
                        seen["x"] = max(seen["x"], x.abs().max().item())
                        seen["w"] = max(seen["w"], w.abs().max().item())
                    return src(x, w, *a, **k)
                return base(x, w, *a, **k)
            return conv
        F.conv2d, F.conv3d = pick(conv2d), pick(conv3d)

    for name in nets:
        setattr(R, name, scoped(name))
    try:
        for size in sizes:
            cfg = shipped_config(size)
            sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
            ocfg = R.config_from_state_dict(sd, size)
            for kind in kinds:
                src, drv = FR.frame(size, 21, kind), FR.frame(size, 22, kind)
                seen = {"x": 0.0, "w": 0.0}
                with torch.no_grad():
                    install(None, None, seen)
                    st0 = R.source_pass(sd, hsd, src, ocfg)
                    img0 = R.driver_pass(sd, hsd, st0, drv, ocfg)
                    tlv0 = st0["target_latent_volume"]
                    print(f"{size}^2 {kind:6s} largest |activation| into a source conv {seen['x']:.2f}, |weight| {seen['w']:.3f}",
                          flush=True)
                    st_fast = None
                    for row, (src_fmt, dec_fmt) in SOURCE_FORMATS.items():
                        install(src_fmt, None)
                        if src_fmt is None:
                            st = st0
                        else:
                            st = st_fast = st_fast or R.source_pass(sd, hsd, src, ocfg)
                        install(None, dec_fmt)
                        img = R.driver_pass(sd, hsd, st, drv, ocfg)
                        install(None, None)
                        err = (img - img0).abs()
                        mse = (err ** 2).mean().item()
                        psnr = 10 * math.log10(1.0 / mse) if mse > 0 else float("inf")
                        u8, u80 = to_u8(img).int(), to_u8(img0).int()
                        changed = (u8 != u80).float().mean().item()
                        levels = (u8 - u80).abs().max().item()
                        e_tlv = (st["target_latent_volume"] - tlv0).abs().max().item()
                        print(f"{size}^2 {kind:6s} {row:36s} image max-abs {err.max().item():.1e} mean-abs {err.mean().item():.1e}  "
                              f"PSNR {psnr:5.1f} dB  uint8 pixels moved {100 * changed:.2f} % (at most {levels} level)  "
                              f"target_latent_volume max-abs {e_tlv:.1e} (of max {tlv0.abs().max().item():.2f})", flush=True)
    finally:
        F.conv2d, F.conv3d = conv2d, conv3d
        for name, fn in nets.items():
            setattr(R, name, fn)


def main():
    if "--source" in sys.argv:
        kinds = [sys.argv[sys.argv.index("--frames") + 1]] if "--frames" in sys.argv else ["smooth", "noise"]
        sizes = [int(a) for a in sys.argv[1:] if a.isdigit()] or [256, 512]
        source_main(sizes, kinds)
        return
    if "--stage2" in sys.argv:
        kinds = [sys.argv[sys.argv.index("--frames") + 1]] if "--frames" in sys.argv else ["smooth", "noise"]
        sizes = [int(a) for a in sys.argv[1:] if a.isdigit()] or [512, 1024]
        stage2_main(sizes, kinds)
        return
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    kind = sys.argv[sys.argv.index("--frames") + 1] if "--frames" in sys.argv else "noise"
    args = [a for a in args if a != kind]
    sizes = [int(a) for a in args] or [256, 512]
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from oracle import frames as FR
    from oracle import restatement as R

    conv2d = F.conv2d
    for size in sizes:
        cfg = shipped_config(size)
        sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
        ocfg = R.config_from_state_dict(sd, size)
        src, drv = FR.frame(size, 21, kind), FR.frame(size, 22, kind)
        with torch.no_grad():
            taps = {}
            R.driver_pass(sd, hsd, R.source_pass(sd, hsd, src, ocfg), drv, ocfg, taps)
            vol = taps["aligned_volume"]
            feat2d = vol.view(vol.shape[0], ocfg.C * ocfg.D, ocfg.S, ocfg.S)
            img0, logits0, _, _ = R.decoder(sd, feat2d)
            for fmt in FORMATS:
                F.conv2d = emulated_conv2d(fmt, conv2d)
                try:
                    img, logits, _, _ = R.decoder(sd, feat2d)
                finally:
                    F.conv2d = conv2d
                err = (img - img0).abs()
                mse = (err ** 2).mean().item()
                psnr = 10 * math.log10(1.0 / mse) if mse > 0 else float("inf")
                changed = (to_u8(img) != to_u8(img0)).float().mean().item()
                print(f"{size}^2 {kind:6s} {fmt:28s} image max-abs {err.max().item():.1e} mean-abs {err.mean().item():.1e}  "
                      f"PSNR {psnr:5.1f} dB  logits max-abs {(logits - logits0).abs().max().item():.1e}  "
                      f"uint8 pixels changed {100 * changed:.1f} %", flush=True)


if __name__ == "__main__":
    main()
