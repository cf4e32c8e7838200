"""CPU emulation behind the error budget of the decoder's one-plane fp16 operand mode (ops.H1, DESIGN.md section 2).

    python tools/decoder_precision_emulation.py [size ...] [--frames noise|smooth]     (default: 256 512, noise)

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


def main():
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
