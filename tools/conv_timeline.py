"""Where does a conv launch spend its time?  (GPU box, instrumented build libemoport_dbg.so.)  One launch with
EMO_CONV_DBG=256 leaves per-CTA %globaltimer stamps of the kernel's phases (conv_igemm.cu: g_conv_stamps); printed here
relative to the earliest CTA entry, as min / median / max over the CTAs, next to the CUDA-event time of the launch.

    python tools/conv_timeline.py --phases

splits each CTA's time over ALL its tiles instead (EMO_CONV_DBG=512, g_conv_phase: SM clock cycles of consumer thread 0 per
phase), for the decoder's multi-tile layers, once as they are and once with the final phase's loads, stores and statistics
switched off (EMO_CONV_DBG bits 4 | 8 | 16; outputs are garbage then)."""
import ctypes as C, math, os, pathlib, sys
ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
os.environ.setdefault("EMO_LIB", str(ROOT / "emoportraits_b200" / "csrc" / "libemoport_dbg.so"))
import numpy as np
import torch
from emoportraits_b200 import lib as L, ops

NAMES = ["entry", "prologue done", "producer starts", "producer done", "first operands landed", "last chunk promoted",
         "final-phase stores issued", "statistics done", "consumer exit"]
dev = "cuda"
g = torch.Generator().manual_seed(0)


def run(Cin, Cout, sp, k, planes, residual=True):
    three = len(sp) == 3
    shape = (1,) + (tuple(sp) if three else (1,) + tuple(sp)) + (Cin,)
    x = torch.randn(shape, generator=g).to(dev)
    w = torch.randn((Cout, Cin) + (k,) * len(sp), generator=g) / math.sqrt(Cin * k ** len(sp))
    pw = ops.pack_conv_weight(w, planes=planes)
    a = ops.split_bf16(x, planes)
    out = torch.empty(shape[:-1] + (Cout,), device=dev)
    res = torch.randn(shape[:-1] + (Cout,), generator=g).to(dev) if residual else None
    ops.begin_pass(dev)
    st = ops.new_stats(1, 32, dev)
    bias = torch.zeros(Cout, device=dev)
    os.environ["EMO_CONV_DBG"] = "0"
    for _ in range(3):
        ops.conv_igemm(a, pw, out=out, bias=bias, residual=res, stats=st)
    torch.cuda.synchronize()
    os.environ["EMO_CONV_DBG"] = "256"
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.conv_igemm(a, pw, out=out, bias=bias, residual=res, stats=st)
    e1.record()
    torch.cuda.synchronize()
    os.environ["EMO_CONV_DBG"] = "0"
    buf = (C.c_ulonglong * (160 * 16))()
    fn = L.load().emo_debug_conv_stamps
    fn.restype = C.c_int
    assert fn(buf) == 0
    s = np.array(buf, dtype=np.uint64).reshape(160, 16).astype(np.float64)
    live = s[:, 0] > 0
    s = s[live]
    t0 = s[:, 0].min()
    print(f"--- {Cin}->{Cout} {sp} k{k} planes {planes}: {int(live.sum())} CTAs, "
          f"launch {e0.elapsed_time(e1) * 1000:.1f} us (events), last stamp {(s[:, :15].max() - t0) / 1000:.1f} us after the first entry")
    for k_, name in enumerate(NAMES):
        col = s[:, k_]
        col = col[col > 0]
        if len(col) == 0:
            continue
        r = (col - t0) / 1000.0
        print(f"    {name:28s} min {r.min():7.2f}  median {np.median(r):7.2f}  max {r.max():7.2f} us   ({len(col)} CTAs)")
    # zero the stamps for the next shape
    return


PHASES = ["operand wait", "main-loop issue", "final loads", "act + stores", "stats + barriers", "tile set-up"]


def sm_clock_mhz():
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return float("nan")


def phases(label, Cin, Cout, sp, k, planes, residual, upconv):
    """residual: 0 none / 1 same resolution / 2 half resolution (as tools/conv_layer_bench.py)"""
    shape = (1, 1) + tuple(sp) + (Cin,)
    x = torch.randn(shape, generator=g).to(dev)
    w = torch.randn((Cout, Cin, k, k), generator=g) / math.sqrt(Cin * k * k)
    a = ops.split_bf16(x, planes)
    osp = tuple(2 * v for v in sp) if upconv else tuple(sp)
    out = torch.empty((1, 1) + osp + (Cout,), device=dev)
    pw = ops.pack_upconv_weight(w) if upconv else ops.pack_conv_weight(w, planes=planes)
    res, rs = None, 0
    if residual == 1:
        res = torch.randn((1, 1) + osp + (Cout,), generator=g).to(dev)
    elif residual == 2:
        res, rs = torch.randn((1, 1, osp[0] // 2, osp[1] // 2, Cout), generator=g).to(dev), 1
    ops.begin_pass(dev)
    st = ops.new_stats(1, 32, dev)
    bias = torch.zeros(Cout, device=dev)
    fn = L.load().emo_debug_conv_phases
    fn.restype = C.c_int
    buf = (C.c_ulonglong * (160 * 8))()
    run = lambda: ops.conv_igemm(a, pw, out=out, bias=bias, residual=res, res_shift=rs, stats=st, upconv=upconv)
    print(f"--- {label}", flush=True)
    for dbg, tag in [(512, "as is"), (512 | 4 | 8 | 16, "no final loads / stores / statistics")]:
        os.environ["EMO_CONV_DBG"] = "0"
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        os.environ["EMO_CONV_DBG"] = str(dbg)
        assert fn(buf, 1) == 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        os.environ["EMO_CONV_DBG"] = "0"
        assert fn(buf, 0) == 0
        s = np.array(buf, dtype=np.uint64).reshape(160, 8).astype(np.float64)
        s = s[s[:, 7] > 0]
        mhz = sm_clock_mhz()
        per_tile = s[:, :6].sum(0) / s[:, 7].sum()  # cycles per tile, over all CTAs
        tot = per_tile.sum()
        cols = "  ".join(f"{n} {c / mhz:6.2f}" for n, c in zip(PHASES, per_tile))
        print(f"    {tag:38s} launch {e0.elapsed_time(e1) * 1000:7.1f} us, {s[:, 7].mean():5.2f} tiles/CTA, "
              f"{tot / mhz:6.2f} us/tile at {mhz:.0f} MHz: {cols}", flush=True)


if len(sys.argv) > 1 and sys.argv[1] == "--phases":
    for args in [("512^2 128->128 conv2+res", 128, 128, (512, 512), 3, 2, 1, False),
                 ("256^2 192->192 conv2+res", 192, 192, (256, 256), 3, 2, 1, False),
                 ("up 256->512 192->128 subpixel", 192, 128, (256, 256), 3, 2, 0, True),
                 ("64^2 512->512 conv2+res", 512, 512, (64, 64), 3, 2, 1, False)]:
        phases(*args)
    sys.exit(0)

run(512, 512, (64, 64), 3, 2)
run(128, 128, (512, 512), 3, 2)
run(320, 320, (128, 128), 3, 2)
run(64, 32, (32, 64, 64), 3, "h2", residual=False)
