"""The case table of the non-convolution kernels, shared by tests/test_op_cases_cpu.py (every case reaches the kernel variant it
names, the table reaches every variant, and every launch the shipped models issue falls in a variant of the table) and
tests/test_op_cases_gpu.py (every case against float64).

A case is one C-ABI call: the entry point, its arguments (`kw`, read by `inputs` / `launch`) and the variant class it reaches.
`classify` restates each entry point's dispatch on the host - which template instantiation, which store path, which capped grid
- from the launch arguments alone, so that it classifies the models' launches (recorded in EMO_DRY_RUN mode) the same way.
Where a branch depends on the device (the grid sampler's brick shape reads the occupancy of its kernel), the restatement uses
an H100 SXM - 132 SMs, 6 resident CTAs per SM as the launch code states - and the cases sit well clear of the threshold."""
from __future__ import annotations

import ctypes as C
import math
import zlib
from dataclasses import dataclass

import torch

import pose_reference as PR

SM_COUNT = 132          # H100 SXM
GS3_CTAS_PER_SM = 6     # gs3_cl_kernel: 40 registers, 18 KB of shared memory (emo_grid_sample3d)
ACT_NAMES = ("none", "relu", "sigmoid", "tanh")
PLANES = {"bf16x2": (2, torch.bfloat16), "bf16x3": (3, torch.bfloat16), "fp16x2": (2, torch.float16), "fp16x1": (1, torch.float16)}
F16_SCALE = 16.0        # ops.F16_ACT_SCALE


@dataclass(frozen=True)
class Case:
    op: str            # C-ABI entry point without the emo_ prefix
    want: str          # variant class (classify)
    kw: tuple          # sorted (name, value) pairs

    @property
    def k(self) -> dict:
        return dict(self.kw)

    @property
    def id(self) -> str:
        return self.op + "-" + "-".join(f"{k}{_fmt(v)}" for k, v in self.kw)


def _fmt(v):
    if isinstance(v, tuple):
        return "x".join(map(str, v)) or "none"
    return str(v)


def case(op, want, **kw) -> Case:
    return Case(op, want, tuple(sorted(kw.items())))


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------------------
# host restatement of the dispatch
# ------------------------------------------------------------------------------------------------------------------
# the arguments of the entry points that take them positionally (the trailing stream excluded)
POSITIONAL = {"emo_gn_stats": ("x", "N", "S", "C", "G", "stats"),
              "emo_maxpool2d_3x3s2": ("x", "N", "H", "W", "C", "out"),
              "emo_global_avgpool": ("x", "N", "S", "C", "out"),
              "emo_split_bf16": ("x", "n", "hi", "lo", "lo2"),
              "emo_split_f16": ("x", "n", "scale", "hi", "lo"),
              "emo_stem_pack": ("x", "N", "H", "W", "C", "scale", "out"),
              "emo_u8_to_image": ("x", "N", "H", "W", "C", "out"),
              "emo_image_to_u8": ("x", "N", "C", "H", "W", "out"),
              "emo_resize_bicubic": ("x", "N", "C", "Hin", "Win", "Hout", "Wout", "out"),
              "emo_composite": ("img", "mask", "bg", "N", "C", "H", "W", "threshold", "out"),
              "emo_parsing_prepare": ("x", "N", "C", "Hin", "Win", "Hout", "Wout", "mean", "std", "out"),
              "emo_parsing_masks": ("x", "N", "K", "Hin", "Win", "Hout", "Wout", "label_sets", "out", "labels"),
              "emo_resize_area": ("x", "N", "C", "Hin", "Win", "Hout", "Wout", "scale", "shift", "out")}
# which of them are device pointers (label_sets is a host array of four class bit sets: a scalar argument)
POSITIONAL_POINTERS = {"x", "stats", "out", "hi", "lo", "lo2", "img", "mask", "bg", "mean", "std", "labels"}


def fields(name: str, args) -> dict:
    """the arguments of one C-ABI call as {field: value}; pointers are ints (0 for NULL)"""
    if args and hasattr(args[0], "_obj"):
        d = args[0]._obj
        return {f: (getattr(d, f) or 0) if t is C.c_void_p else getattr(d, f) for f, t in d._fields_}
    out = {}
    for k, v in zip(POSITIONAL[name], args):
        if isinstance(v, C.Array):
            out[k] = list(v)
        else:
            out[k] = (v.value if hasattr(v, "value") else v) or 0
    return out


def pointer_fields(name: str, args) -> set:
    """the names of the pointer arguments of one C-ABI call (NULL or not)"""
    if args and hasattr(args[0], "_obj"):
        return {f for f, t in args[0]._obj._fields_ if t is C.c_void_p}
    return set(POSITIONAL[name]) & POSITIONAL_POINTERS


def _outs(f, fp16_key="plane_fp16"):
    """output format of an apply / grid-sampler call: fp32 and / or operand planes"""
    o = ["fp32"] if f["out"] else []
    if f["out_hi"]:
        if f[fp16_key]:
            o.append("fp16x2" if f["out_lo"] else "fp16x1")
        else:
            o.append("bf16x3" if f["out_lo2"] else "bf16x2")
    return "+".join(o)


def apply_grid(f):
    """(V, blocks per sample, cv_step) of emo_apply"""
    V = 2 if f["C"] % 8 == 0 else 1
    cvn = f["C"] // (4 * V)
    per_n = f["D"] * f["H"] * f["W"] * cvn
    blocks = max(1, min(cdiv(per_n, 256), (SM_COUNT * 32) // max(f["N"], 1)))
    return V, per_n, blocks, (blocks * 256) % cvn


def gs3_brick(f):
    """brick (bw, bh, bd) of the channels-last grid sampler and whether its height was halved (emo_grid_sample3d)"""
    N, Do, Ho, Wo = f["N"], f["Dout"], f["Hout"], f["Wout"]
    slots = SM_COUNT * GS3_CTAS_PER_SM
    bw, bh, bd = min(8, Wo), min(8, Ho), min(2, Do)
    ctas = lambda: N * cdiv(Wo, bw) * cdiv(Ho, bh) * cdiv(Do, bd)  # noqa: E731
    if ctas() < 4 * slots:
        if Do >= 4 and Ho >= 4 and Wo >= 4:
            bw, bh, bd = 4, 4, 4
        else:
            bd = 1
    h0 = bh
    while ctas() < 4 * SM_COUNT and bh > 2:
        bh >>= 1
    return (bw, bh, bd), bh != h0, ctas()


def resample_grid(f, pooled):
    """(blocks per sample, fixed_c) of emo_upsample_trilinear / emo_avgpool"""
    if pooled:
        per_n = (f["D"] // f["fd"]) * (f["H"] // f["fh"]) * (f["W"] // f["fw"]) * (f["C"] // 4)
    else:
        per_n = f["D"] * f["fd"] * f["H"] * f["fh"] * f["W"] * f["fw"] * (f["C"] // 4)
    bx = max(1, min(cdiv(per_n, 1024), SM_COUNT * 16))
    return bx, (bx * 256) % (f["C"] // 4) == 0


def classify(name: str, f: dict):
    """(variant class, set of finer features) of one C-ABI call"""
    op = name[4:]
    feats = set()
    if op == "apply":
        V, per_n, blocks, cv_step = apply_grid(f)
        inst = f"apply<{f['up']},{V},{'f16' if f['plane_fp16'] else 'bf16'}>"
        src = ("gn+ada" if f["ada_w"] else "gn") if f["stats"] else ("AB[n]" if f["ab_per_sample"] else "AB") if f["A"] else "none"
        res = ("res+A2B2" if f["A2"] else "res") if f["res"] else "nores"
        out = _outs(f)
        feats |= {inst, f"affine {src}", f"residual {res}", f"act {ACT_NAMES[f['act']]}", f"out {out}"}
        if f["up"] == 2 and f["D"] > 1:
            feats.add("up=2 with D > 1")
        if f["N"] > 1:
            feats.add("N > 1")
        if per_n > blocks * 256:
            feats.add("grid-stride loop, cv_step != 0" if cv_step else "grid-stride loop, cv_step == 0")
        return f"{inst} {out}", feats
    if op == "gn_stats":
        c4n, N = f["C"] // 4, f["N"]
        L = min(c4n, 256)
        chunks = max(1, f["S"] * c4n // 4096)
        cap = max(1, (SM_COUNT * 8) // N)
        rows = "channel loop (C/4 > 256)" if c4n > 256 else "idle row slots" if 256 % L else "all row slots"
        feats |= {rows, f"cpg {f['C'] // f['G']}", f"N {N}",
                  "capped chunks" if chunks > cap else "one chunk" if chunks == 1 else "several chunks"}
        return f"gn_stats {rows}", feats
    if op == "gn_finalize":
        kind = "adaptive" if f["ada_w"] else "plain"
        feats |= {kind} | ({"N > 1"} if f["N"] > 1 else set())
        return f"gn_finalize {kind}", feats
    if op == "gn_head":
        feats |= {f"Cout {f['Cout']}"}
        feats |= {"C % 128 != 0"} if f["C"] % 128 else set()
        feats |= {"S % 8 != 0"} if f["S"] % 8 else set()
        feats |= {"N > 1"} if f["N"] > 1 else set()
        return "gn_head", feats
    if op == "grid_sample3d":
        out = _outs(f)
        coord = "theta" if f["theta"] else "grid"
        if f["in_layout"] == 0:
            feats |= {f"ncdhw {out}", f"ncdhw {coord}"}
            return f"gs3_nc {out}", feats
        store = "vector" if f["os_c"] == 1 else "strided"
        (bw, bh, bd), halved, _ = gs3_brick(f)
        brick = "4x4x4" if bd == 4 else f"8x8x{bd}" if (bw, bh) == (min(8, f["Wout"]), min(8, f["Hout"])) or halved else "?"
        feats |= {f"cl {out} {store} {coord}", f"brick {brick}" if not halved else "brick height halved",
                  f"{store} stores"}
        for ax, nm in (("Dout", "D"), ("Wout", "W")):
            if f[ax] == 1:
                feats.add(f"{nm} = 1 lattice")
        if f["Wout"] % bw or f["Hout"] % bh or f["Dout"] % bd:
            feats.add("ragged bricks")
        return f"gs3_cl<{'split' if f['out_hi'] else 'fp32'}> {out} {store}", feats
    if op in ("upsample_trilinear", "avgpool"):
        bx, fixed = resample_grid(f, op == "avgpool")
        fac = f"({f['fd']},{f['fh']},{f['fw']})"
        feats |= {f"{op} f={fac}"}
        if f["stats"]:
            feats.add(f"{op} stats {'fixed_c' if fixed else 'per-element'}")
            feats |= {f"{op} stats N > 1"} if f["N"] > 1 else set()
        if f["add"]:
            feats.add(f"{op} add")
        return f"{op}{' stats' if f['stats'] else ''}", feats
    if op == "linear":
        K = f["K"]
        if f["xs_k"] != 1 or f["xs_m"] != K:
            feats.add("strided x")
        if f["os_n"] != 1 or f["os_m"] != f["N"]:
            feats.add("strided out")
        feats |= {"K < 32"} if K < 32 else {"K % 32 != 0"} if K % 32 else {"K % 32 == 0"}
        feats |= {"add"} if f["add"] else set()
        feats |= {"scale != 1"} if f["scale"] != 1.0 else set()
        feats |= {f"act {ACT_NAMES[f['act']]}"}
        return "linear", feats
    if op == "conv_direct":
        feats |= {f"stride {f['stride']}"}
        feats |= {"Cout = 4 x odd"} if (f["Cout"] // 4) % 2 else set()
        if f["stats"]:
            feats |= {"stats"} | ({"stats N > 1"} if f["N"] > 1 else set())
        return f"conv_direct s{f['stride']}{' stats' if f['stats'] else ''}", feats
    if op == "maxpool2d_3x3s2":
        feats |= {f"H {'odd' if f['H'] % 2 else 'even'}", f"W {'odd' if f['W'] % 2 else 'even'}"}
        return "maxpool2d_3x3s2", feats
    if op == "global_avgpool":
        feats |= {"S >= 256^2"} if f["S"] >= 256 * 256 else set()
        return "global_avgpool", feats
    if op in ("resize_bilinear", "grid_sample2d_affine"):
        if f["C_pad"] > f["C"]:
            feats.add("C_pad > C zero fill")
        if f["mean"]:
            feats.add("mean/std")
        if op == "resize_bilinear":
            hi, wi, ho, wo = f["Hin"], f["Win"], f["Hout"], f["Wout"]
            if (hi, wi) == (ho, wo):
                feats.add("same size")
            elif ho > hi or wo > wi:
                feats.add("up")
            else:
                feats.add("down")
            if (hi % ho and ho % hi) or (wi % wo and wo % wi):
                feats.add("non-integer ratio")
        elif f["out_nchw"]:
            feats.add("NCHW copy")
        return op, feats
    if op in ("split_bf16", "split_f16"):
        n = (3 if f["lo2"] else 2) if op == "split_bf16" else (2 if f["lo"] else 1)
        return f"{op} x{n}", {f"{op} x{n}"}
    if op == "stem_pack":
        feats.add("stem_pack")
        if f["N"] * f["H"] * f["W"] > STRIDE_CAP * 256:
            feats.add("stem_pack grid-stride loop")
        return op, feats
    if op == "pose_theta":
        inp = "theta_in" if f["theta_in"] else "srt"
        mix = ("mix_old" if f["mix_old"] else "mix") if f["mix"] else "nomix"
        smooth = bool(f["smooth_state"])
        cls = f"pose_theta {inp} {mix}{' smooth' if smooth else ''}"
        inv = "invert" if f["invert_warp"] else "no invert"
        feats |= {cls, f"pose {inp} {mix} {inv}", inv, "align" if f["align2d"] else "no align"}
        if smooth:
            start = "init" if f["smooth_init"] else "carried"
            feats |= {f"smooth {start}", f"momentum {f['smooth_momentum']:.6g} {start}"}
            if f["N"] > 1:
                feats.add("one-thread walk")     # smoothing: one thread walks the samples in order
        if f["N"] > 32:
            feats.add("N > 32")                  # 32 threads per block
        return cls, feats
    if op in BOUNDARY_GRID:
        # the wrapper-boundary kernels (tests/model_op_launches.py BOUNDARY): capped grid-stride loops
        work = {"u8_to_image": ("N", "H", "W"), "image_to_u8": ("N", "H", "W"), "composite": ("N", "C", "H", "W"),
                "resize_bicubic": ("N", "C", "Hout", "Wout"), "parsing_prepare": ("N", "C", "Hout", "Wout"),
                "parsing_masks": ("N", "Hout", "Wout"), "resize_area": ("N", "C", "Hout", "Wout")}[op]
        blocks, threads = BOUNDARY_GRID[op]
        if math.prod(f[k] for k in work) > blocks * threads:
            feats.add(f"{op} grid-stride loop")
        if "Hin" in f:
            hi, wi, ho, wo = f["Hin"], f["Win"], f["Hout"], f["Wout"]
            feats.add(f"{op} {'same size' if (hi, wi) == (ho, wo) else 'up' if ho > hi or wo > wi else 'down'}")
        return op, feats
    raise KeyError(name)


STRIDE_CAP = SM_COUNT * 16   # CTAs of the capped grid-stride loops (emo_stem_pack, the image conversions, the composite)
# (CTAs, threads per CTA) of each wrapper-boundary kernel's capped grid
BOUNDARY_GRID = {"u8_to_image": (STRIDE_CAP, 256), "image_to_u8": (STRIDE_CAP, 256), "composite": (STRIDE_CAP, 256),
                 "resize_bicubic": (STRIDE_CAP, 256), "parsing_prepare": (STRIDE_CAP, 256),
                 "parsing_masks": (SM_COUNT * 32, 128), "resize_area": (STRIDE_CAP, 256)}


# ------------------------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------------------------
A, BF2, BF3, H2, H1 = "AB", "bf16x2", "bf16x3", "fp16x2", "fp16x1"
CASES = [
    # ---- emo_apply: 8 instantiations x affine source x residual x act x output format ----
    case("apply", up=1, want="apply<1,2,bf16> bf16x2", N=1, C=64, sp=(1, 24, 40), src="gn", res="res", act=1, out=(BF2,)),
    case("apply", up=1, want="apply<1,2,bf16> fp32+bf16x3", N=2, C=96, sp=(4, 12, 20), src="gn+ada", res="nores", act=3, out=("fp32", BF3)),
    case("apply", up=1, want="apply<1,2,bf16> fp32", N=1, C=32, sp=(1, 16, 16), src="none", res="res+A2B2", act=2, out=("fp32",)),
    case("apply", up=1, want="apply<1,1,bf16> fp32+bf16x2", N=2, C=20, sp=(1, 12, 36), src="AB[n]", res="res", act=0, out=("fp32", BF2)),
    case("apply", up=1, want="apply<1,1,bf16> fp32", N=1, C=20, sp=(1, 512, 512), src="AB", res="nores", act=1, out=("fp32",)),
    case("apply", up=1, want="apply<1,1,bf16> bf16x3", N=1, C=12, sp=(3, 8, 8), src="gn+ada", res="res", act=2, out=(BF3,)),
    case("apply", up=2, want="apply<2,2,bf16> fp32+bf16x2", N=2, C=64, sp=(3, 10, 14), src="gn+ada", res="res+A2B2", act=1, out=("fp32", BF2)),
    case("apply", up=2, want="apply<2,2,bf16> bf16x2", N=1, C=64, sp=(1, 16, 16), src="gn", res="nores", act=1, out=(BF2,)),
    case("apply", up=2, want="apply<2,2,bf16> bf16x3", N=1, C=40, sp=(1, 16, 12), src="AB", res="nores", act=3, out=(BF3,)),
    case("apply", up=2, want="apply<2,1,bf16> fp32", N=1, C=36, sp=(2, 9, 7), src="gn", res="res", act=0, out=("fp32",)),
    case("apply", up=2, want="apply<2,1,bf16> bf16x2", N=2, C=12, sp=(1, 8, 6), src="AB[n]", res="res+A2B2", act=3, out=(BF2,)),
    case("apply", up=1, want="apply<1,2,f16> fp16x2", N=1, C=128, sp=(1, 32, 32), src="gn", res="nores", act=1, out=(H2,)),
    case("apply", up=1, want="apply<1,2,f16> fp16x1", N=1, C=64, sp=(2, 16, 16), src="gn+ada", res="res", act=1, out=(H1,)),
    case("apply", up=1, want="apply<1,2,f16> fp32+fp16x2", N=2, C=48, sp=(1, 20, 20), src="AB[n]", res="res+A2B2", act=2, out=("fp32", H2)),
    case("apply", up=1, want="apply<1,1,f16> fp32+fp16x1", N=1, C=28, sp=(1, 10, 30), src="gn", res="nores", act=3, out=("fp32", H1)),
    case("apply", up=1, want="apply<1,1,f16> fp16x2", N=2, C=4, sp=(2, 6, 10), src="none", res="res", act=1, out=(H2,)),
    case("apply", up=2, want="apply<2,2,f16> fp16x1", N=1, C=64, sp=(1, 16, 16), src="gn", res="nores", act=1, out=(H1,)),
    case("apply", up=2, want="apply<2,2,f16> fp32+fp16x2", N=2, C=32, sp=(2, 6, 8), src="AB", res="res", act=0, out=("fp32", H2)),
    case("apply", up=2, want="apply<2,1,f16> fp16x2", N=1, C=20, sp=(2, 7, 9), src="gn+ada", res="res+A2B2", act=2, out=(H2,)),
    case("apply", up=2, want="apply<2,1,f16> fp16x1", N=2, C=4, sp=(1, 5, 11), src="AB[n]", res="nores", act=1, out=(H1,)),
    # ---- emo_gn_stats ----
    case("gn_stats", "gn_stats idle row slots", N=1, C=96, G=32, sp=(1, 40, 40)),
    case("gn_stats", "gn_stats all row slots", N=2, C=128, G=32, sp=(1, 3, 5)),
    case("gn_stats", "gn_stats channel loop (C/4 > 256)", N=2, C=1536, G=32, sp=(1, 30, 30)),
    case("gn_stats", "gn_stats all row slots", N=5, C=64, G=64, sp=(1, 256, 256)),
    case("gn_stats", "gn_stats idle row slots", N=1, C=48, G=16, sp=(2, 64, 64)),
    case("gn_stats", "gn_stats all row slots", N=2, C=512, G=32, sp=(1, 64, 64)),
    # ---- emo_gn_finalize / emo_gn_head ----
    case("gn_finalize", "gn_finalize plain", N=3, C=96, G=32, ada=False),
    case("gn_finalize", "gn_finalize adaptive", N=2, C=64, G=16, ada=True),
    case("gn_head", "gn_head", N=2, C=96, sp=(1, 13, 7), Cout=1, act=2),
    case("gn_head", "gn_head", N=2, C=160, sp=(1, 9, 11), Cout=2, act=0),
    case("gn_head", "gn_head", N=2, C=64, sp=(1, 15, 15), Cout=4, act=3),
    case("gn_head", "gn_head", N=1, C=256, sp=(1, 20, 20), Cout=3, act=2),
]


def _gs3(want, N, C, ins, outs, layout="cl", out_layout="cl", f32=True, planes=None, coord="grid"):
    return case("grid_sample3d", want, N=N, C=C, ins=ins, outs=outs, layout=layout, out_layout=out_layout, f32=f32,
                planes=planes or "none", coord=coord)


CASES += [
    # channels-last kernel: {fp32, +bf16x2, +bf16x3, fp16x1 alone} x {vector, strided stores} x {grid, theta} over the brick branches
    _gs3("gs3_cl<fp32> fp32 vector", 1, 4, (32, 48, 48), (128, 128, 128)),                                     # 8x8x2
    _gs3("gs3_cl<fp32> fp32 vector", 1, 8, (16, 16, 16), (40, 48, 48), out_layout="hwdc", coord="theta"),      # 4x4x4
    _gs3("gs3_cl<fp32> fp32 strided", 2, 12, (8, 12, 10), (3, 160, 160), out_layout="ncdhw"),                  # 8x8x1
    _gs3("gs3_cl<fp32> fp32 strided", 1, 8, (6, 20, 20), (1, 24, 1), out_layout="ncdhw", coord="theta"),       # halved, D = W = 1
    _gs3("gs3_cl<split> fp32+bf16x2 vector", 2, 16, (5, 7, 9), (5, 7, 9), planes=BF2),                            # halved, ragged
    _gs3("gs3_cl<split> fp32+bf16x2 vector", 1, 8, (16, 16, 16), (40, 48, 48), planes=BF2, coord="theta"),
    _gs3("gs3_cl<split> fp32+bf16x2 strided", 1, 8, (8, 12, 10), (3, 160, 160), out_layout="ncdhw", planes=BF2),
    _gs3("gs3_cl<split> fp32+bf16x2 strided", 2, 4, (5, 7, 9), (5, 7, 9), out_layout="ncdhw", planes=BF2, coord="theta"),
    _gs3("gs3_cl<split> bf16x2 vector", 1, 16, (16, 32, 32), (16, 32, 32), out_layout="hwdc", f32=False, planes=BF2, coord="theta"),
    _gs3("gs3_cl<split> fp32+bf16x3 vector", 1, 4, (32, 48, 48), (128, 128, 128), planes=BF3),
    _gs3("gs3_cl<split> fp32+bf16x3 vector", 2, 8, (4, 9, 9), (1, 17, 23), out_layout="hwdc", planes=BF3, coord="theta"),
    _gs3("gs3_cl<split> fp32+bf16x3 strided", 1, 8, (16, 16, 16), (40, 48, 48), out_layout="ncdhw", planes=BF3),
    _gs3("gs3_cl<split> fp32+bf16x3 strided", 1, 12, (8, 12, 10), (3, 160, 160), out_layout="ncdhw", planes=BF3, coord="theta"),
    _gs3("gs3_cl<split> fp16x1 vector", 1, 8, (8, 12, 10), (3, 160, 160), f32=False, planes=H1),
    _gs3("gs3_cl<split> fp16x1 vector", 1, 4, (32, 48, 48), (128, 128, 128), f32=False, planes=H1, coord="theta"),
    _gs3("gs3_cl<split> fp16x1 strided", 1, 8, (16, 16, 16), (40, 48, 48), out_layout="ncdhw", f32=False, planes=H1),
    _gs3("gs3_cl<split> fp16x1 strided", 2, 4, (6, 20, 20), (4, 1, 24), out_layout="ncdhw", f32=False, planes=H1, coord="theta"),
    # boundary grid: points at +-1, on voxel centres, less than one voxel outside and far outside
    _gs3("gs3_cl<fp32> fp32 vector", 1, 8, (8, 16, 32), (6, 16, 16), coord="boundary"),
    _gs3("gs3_nc fp32", 1, 8, (8, 16, 32), (6, 16, 16), layout="ncdhw", out_layout="ncdhw", coord="boundary"),
    # NCDHW kernel with and without planes
    _gs3("gs3_nc fp32", 2, 5, (6, 9, 11), (4, 7, 1), layout="ncdhw", out_layout="ncdhw", coord="theta"),
    _gs3("gs3_nc fp32+bf16x2", 1, 6, (6, 9, 11), (1, 10, 12), layout="ncdhw", out_layout="ncdhw", planes=BF2),
    _gs3("gs3_nc fp32+bf16x3", 2, 3, (5, 8, 8), (5, 8, 8), layout="ncdhw", out_layout="ncdhw", planes=BF3, coord="theta"),
    _gs3("gs3_nc fp16x1", 1, 4, (5, 8, 8), (3, 5, 6), layout="ncdhw", out_layout="ncdhw", f32=False, planes=H1),
]

_F8 = [(a, b, c) for a in (1, 2) for b in (1, 2) for c in (1, 2)]
CASES += [case("upsample_trilinear", "upsample_trilinear" + (" stats" if i % 2 == 0 else ""), N=2 if i % 3 else 1,
               C=(64, 96, 96, 32, 64, 8, 96, 128)[i], sp=(3, 5, 6), f=f, add=i in (1, 4, 6), stats=i % 2 == 0)
          for i, f in enumerate(_F8)]
CASES += [case("avgpool", "avgpool" + (" stats" if i % 2 == 1 else ""), N=2 if i % 3 != 1 else 1,
               C=(64, 96, 32, 96, 64, 8, 96, 128)[i], sp=(4, 6, 8), f=f, add=i in (0, 3, 5), stats=i % 2 == 1)
          for i, f in enumerate(_F8)]
CASES += [
    # fixed_c branch on a capped grid (bx = 2112 blocks: 2112 * 256 % 24 == 0) - the branch the model's C = 96 volumes take
    case("upsample_trilinear", "upsample_trilinear stats", N=1, C=96, sp=(16, 64, 64), f=(2, 2, 2), add=True, stats=True),
    case("avgpool", "avgpool stats", N=2, C=96, sp=(32, 64, 64), f=(1, 2, 2), add=False, stats=True),
    # ---- emo_linear: the model's strided operands (nets.py), K < 32, K % 32 != 0, add + scale + act ----
    case("linear", "linear", M=40, N=24, K=16, xs=(16, 1), os=(1, 40), bias=False, add=False, scale=1.0, act=0),
    case("linear", "linear", M=37, N=70, K=50, xs=(1, 37), os=(1, 37), bias=True, add=True, scale=0.5, act=1),
    case("linear", "linear", M=3, N=9, K=512, xs=(512, 1), os=(9, 1), bias=True, add=False, scale=1.0, act=0),
    case("linear", "linear", M=64, N=5, K=7, xs=(7, 1), os=(1, 64), bias=True, add=True, scale=2.0, act=3),
    case("linear", "linear", M=16, N=33, K=45, xs=(1, 16), os=(33, 1), bias=False, add=True, scale=1.0, act=2),
    # ---- emo_conv_direct ----
    case("conv_direct", "conv_direct s1 stats", N=2, sp=(32, 32), cin=4, Cout=64, k=7, stride=1, stats=True, G=32),
    case("conv_direct", "conv_direct s2 stats", N=2, sp=(32, 32), cin=4, Cout=64, k=7, stride=2, stats=True, G=16),
    case("conv_direct", "conv_direct s1", N=1, sp=(13, 17), cin=4, Cout=12, k=3, stride=1, stats=False, G=0),
    case("conv_direct", "conv_direct s2", N=2, sp=(15, 9), cin=8, Cout=20, k=7, stride=2, stats=False, G=0),
    case("conv_direct", "conv_direct s1 stats", N=2, sp=(16, 16), cin=4, Cout=4, k=3, stride=1, stats=True, G=2),
    # ---- emo_maxpool2d_3x3s2 / emo_global_avgpool ----
    case("maxpool2d_3x3s2", "maxpool2d_3x3s2", N=2, H=17, W=16, C=64, neg=False),
    case("maxpool2d_3x3s2", "maxpool2d_3x3s2", N=1, H=16, W=21, C=12, neg=True),
    case("maxpool2d_3x3s2", "maxpool2d_3x3s2", N=2, H=9, W=7, C=8, neg=True),
    case("global_avgpool", "global_avgpool", N=2, S=256 * 256, C=4),
    case("global_avgpool", "global_avgpool", N=3, S=37, C=100),
    # ---- emo_resize_bilinear / emo_grid_sample2d_affine ----
    case("resize_bilinear", "resize_bilinear", N=2, C=3, ins=(64, 48), outs=(64, 48), C_pad=4, norm=False),
    case("resize_bilinear", "resize_bilinear", N=1, C=3, ins=(50, 70), outs=(50, 70), C_pad=8, norm=False),
    case("resize_bilinear", "resize_bilinear", N=2, C=3, ins=(20, 30), outs=(64, 48), C_pad=4, norm=True),
    case("resize_bilinear", "resize_bilinear", N=1, C=3, ins=(100, 90), outs=(37, 41), C_pad=4, norm=True),
    case("resize_bilinear", "resize_bilinear", N=1, C=4, ins=(96, 96), outs=(32, 32), C_pad=4, norm=False),
    case("grid_sample2d_affine", "grid_sample2d_affine", N=2, C=3, ins=(40, 56), outs=(24, 20), C_pad=4, norm=True, nchw=True),
    case("grid_sample2d_affine", "grid_sample2d_affine", N=1, C=3, ins=(33, 31), outs=(16, 16), C_pad=8, norm=False, nchw=False),
    # ---- emo_split_bf16 / emo_split_f16 ----
    case("split_bf16", "split_bf16 x2", n=4 * 10007, planes=2),
    case("split_bf16", "split_bf16 x3", n=4 * 10007, planes=3),
    case("split_f16", "split_f16 x2", n=4 * 10007, planes=2),
    case("split_f16", "split_f16 x1", n=4 * 10007, planes=1),
    # ---- emo_stem_pack: one pass, and the capped grid's stride loop (768 x 720 pixels > 2112 CTAs x 256) ----
    case("stem_pack", "stem_pack", N=2, H=37, W=53),
    case("stem_pack", "stem_pack", N=1, H=768, W=720),
]


def _pose(want, src, mix, invert, align, N, angles="inside", smooth=None, init=False):
    """an emo_pose_theta case: src "srt" (angles "inside" the [-pi/2, pi] clamp, "beyond" it, or at its "edges") or
    "theta_in" (a sheared affine); with smooth (the momentum), a call that seeds the state (init) or carries a seeded one"""
    kw = dict(src=src, mix=mix, invert=invert, align=align, N=N, angles=angles if src == "srt" else "none")
    if smooth is not None:
        kw.update(smooth=smooth, init=init)
    return case("pose_theta", want, **kw)


CASES += [
    # ---- emo_pose_theta: input x mix x invert, align2d set and NULL, one block and several ----
    _pose("pose_theta srt nomix", "srt", "nomix", True, True, 1),
    _pose("pose_theta srt nomix", "srt", "nomix", False, False, 32, "beyond"),
    _pose("pose_theta srt mix", "srt", "mix", True, False, 33, "edges"),
    _pose("pose_theta srt mix", "srt", "mix", False, True, 300),
    _pose("pose_theta srt mix_old", "srt", "mix_old", True, True, 1, "beyond"),
    _pose("pose_theta srt mix_old", "srt", "mix_old", False, False, 33, "edges"),
    _pose("pose_theta theta_in nomix", "theta_in", "nomix", True, False, 300),
    _pose("pose_theta theta_in nomix", "theta_in", "nomix", False, True, 1),
    _pose("pose_theta theta_in mix", "theta_in", "mix", True, True, 32),
    _pose("pose_theta theta_in mix", "theta_in", "mix", False, False, 33),
    _pose("pose_theta theta_in mix_old", "theta_in", "mix_old", True, False, 1),
    _pose("pose_theta theta_in mix_old", "theta_in", "mix_old", False, True, 300, "beyond"),
    # smoothing: per momentum a call that seeds the state and one that carries a seeded state
    _pose("pose_theta srt mix smooth", "srt", "mix", False, True, 3, smooth=0.5, init=True),
    _pose("pose_theta srt mix smooth", "srt", "mix", True, False, 33, smooth=0.5),
    _pose("pose_theta theta_in nomix smooth", "theta_in", "nomix", False, True, 1, smooth=0.3, init=True),
    _pose("pose_theta theta_in nomix smooth", "theta_in", "nomix", False, False, 33, smooth=0.3),
    _pose("pose_theta srt mix_old smooth", "srt", "mix_old", True, True, 4, smooth=0.9, init=True),
    _pose("pose_theta theta_in nomix smooth", "theta_in", "nomix", False, True, 5, smooth=0.9),
    _pose("pose_theta theta_in mix smooth", "theta_in", "mix", False, False, 2, smooth=0.6, init=True),
    _pose("pose_theta srt nomix smooth", "srt", "nomix", True, True, 300, "beyond", smooth=0.6),
    _pose("pose_theta srt nomix smooth", "srt", "nomix", False, True, 3, "beyond", smooth=0.99, init=True),
    _pose("pose_theta theta_in mix_old smooth", "theta_in", "mix_old", False, True, 33, smooth=0.99),
    _pose("pose_theta theta_in mix_old smooth", "theta_in", "mix_old", True, True, 5, smooth=0.01, init=True),
    _pose("pose_theta srt mix smooth", "srt", "mix", False, False, 300, smooth=0.01),
    _pose("pose_theta srt nomix smooth", "srt", "nomix", True, False, 2, smooth=0.0, init=True),
    _pose("pose_theta theta_in mix smooth", "theta_in", "mix", True, True, 32, smooth=0.0),
    _pose("pose_theta theta_in nomix smooth", "theta_in", "nomix", False, True, 3, smooth=1.0, init=True),
    _pose("pose_theta srt mix_old smooth", "srt", "mix_old", False, False, 2, "edges", smooth=1.0),
]
POSE_MOMENTA = (0.5, 0.3, 0.9, 0.6, 0.99, 0.01, 0.0, 1.0)


# C-ABI entry points outside the table: the convolution (tests/conv_plan_cases.py), the wrapper-boundary image conversions
# and mask kernels (tests/test_ops_gpu.py, tests/test_masks.py, and at the wrappers' shapes the BOUNDARY launches of
# tests/model_op_launches.py) and the benchmark's L2 flush
NOT_IN_TABLE = ("conv_igemm", "u8_to_image", "image_to_u8", "resize_bicubic", "composite", "parsing_prepare",
                "parsing_masks", "resize_area", "l2_flush", "l2_flush_clean")


# tags a case carries that the launch arguments do not show (its data)
def tags(c: Case) -> set:
    k = c.k
    t = set()
    if c.op == "grid_sample3d" and k["coord"] == "boundary":
        t.add(f"boundary grid, {'cl' if k['layout'] == 'cl' else 'ncdhw'}")
    if c.op == "maxpool2d_3x3s2" and k["neg"]:
        t.add("all-negative input")
    if c.op == "grid_sample2d_affine":
        t.add("lattice partly outside")
    if c.op == "pose_theta":
        t.add({"inside": "angles inside the clamp", "beyond": "angles beyond the clamp", "edges": "angles at -pi/2 and pi",
               "none": "sheared affine theta_in"}[k["angles"]])
    return t


# every variant of the non-convolution kernels that the table must reach
def required() -> list:
    req = [f"apply<{u},{v},{p}>" for u in (1, 2) for v in (1, 2) for p in ("bf16", "f16")]
    req += [f"affine {s}" for s in ("none", "AB", "AB[n]", "gn", "gn+ada")]
    req += [f"residual {r}" for r in ("nores", "res", "res+A2B2")]
    req += [f"act {a}" for a in ACT_NAMES]
    req += [f"out {o}" for o in ("fp32", "bf16x2", "fp32+bf16x2", "bf16x3", "fp32+bf16x3", "fp16x2", "fp32+fp16x2", "fp16x1",
                                  "fp32+fp16x1")]
    req += ["up=2 with D > 1", "N > 1", "grid-stride loop, cv_step != 0"]
    req += ["idle row slots", "all row slots", "channel loop (C/4 > 256)", "cpg 1", "cpg 3", "cpg 4", "cpg 16", "one chunk",
            "several chunks", "capped chunks", "N 1", "N 2", "N 5"]
    req += ["plain", "adaptive"]
    req += ["Cout 1", "Cout 2", "Cout 3", "Cout 4", "C % 128 != 0", "S % 8 != 0"]
    req += [f"cl {o} {s} {g}" for o in ("fp32", "fp32+bf16x2", "fp32+bf16x3", "fp16x1") for s in ("vector", "strided")
            for g in ("grid", "theta")]
    req += [f"brick {b}" for b in ("8x8x2", "4x4x4", "8x8x1")] + ["brick height halved", "vector stores", "strided stores"]
    req += ["D = 1 lattice", "W = 1 lattice", "ragged bricks", "boundary grid, cl", "boundary grid, ncdhw"]
    req += ["ncdhw fp32", "ncdhw fp32+bf16x2", "ncdhw fp32+bf16x3", "ncdhw fp16x1", "ncdhw grid", "ncdhw theta"]
    for op in ("upsample_trilinear", "avgpool"):
        req += [f"{op} f=({a},{b},{c})" for a, b, c in _F8]
        req += [f"{op} add", f"{op} stats fixed_c", f"{op} stats per-element", f"{op} stats N > 1"]
    req += ["strided x", "strided out", "K < 32", "K % 32 != 0", "add", "scale != 1"]
    req += ["stride 1", "stride 2", "Cout = 4 x odd", "stats", "stats N > 1"]
    req += ["H odd", "H even", "W odd", "W even", "all-negative input", "S >= 256^2"]
    req += ["same size", "up", "down", "non-integer ratio", "C_pad > C zero fill", "mean/std", "lattice partly outside", "NCHW copy"]
    req += ["split_bf16 x2", "split_bf16 x3", "split_f16 x2", "split_f16 x1"]
    req += ["stem_pack", "stem_pack grid-stride loop"]
    pose = [(i, m) for i in ("srt", "theta_in") for m in ("nomix", "mix", "mix_old")]
    req += [f"pose {i} {m} {v}" for i, m in pose for v in ("invert", "no invert")] + [f"pose_theta {i} {m} smooth" for i, m in pose]
    req += ["invert", "no invert", "align", "no align", "smooth init", "smooth carried", "N > 32", "one-thread walk"]
    req += [f"momentum {m:g} {s}" for m in POSE_MOMENTA for s in ("init", "carried")]
    req += ["angles inside the clamp", "angles beyond the clamp", "angles at -pi/2 and pi", "sheared affine theta_in"]
    return req


# ------------------------------------------------------------------------------------------------------------------
# operands and launches
# ------------------------------------------------------------------------------------------------------------------
def gen(c: Case):
    return torch.Generator().manual_seed(zlib.crc32(c.id.encode()))


def gs3_grid(c: Case, g):
    """the sample points (N, Do, Ho, Wo, 3) of a grid case"""
    k = c.k
    N, (Do, Ho, Wo) = k["N"], k["outs"]
    if k["coord"] == "boundary":
        # per axis: +-1, voxel centres, within one voxel outside [-1, 1], far outside, plus a few interior points
        vals = []
        for n in (k["ins"][2], k["ins"][1], k["ins"][0]):    # x, y, z
            cen = [(2 * i + 1) / n - 1 for i in range(n)]
            vals.append(torch.tensor([-1.0, 1.0, -1 - 0.4 / n, 1 + 0.4 / n, -1 - 1.6 / n, 1 + 1.9 / n, -3.0, 2.5, 0.3] + cen))
        idx = [torch.randint(0, len(v), (N, Do, Ho, Wo), generator=g) for v in vals]
        return torch.stack([v[i] for v, i in zip(vals, idx)], -1).float().contiguous()
    zs, ys, xs = (torch.linspace(-1, 1, n) for n in (Do, Ho, Wo))
    w, v, u = torch.meshgrid(zs, ys, xs, indexing="ij")
    base = torch.stack([u, v, w], -1)[None].repeat(N, 1, 1, 1, 1)
    return (1.1 * base + 0.15 * torch.randn(base.shape, generator=g) + 0.05).contiguous()


def gs3_theta(c: Case, g):
    N = c.k["N"]
    th = torch.zeros(N, 3, 4)
    for n in range(N):
        a = 0.3 + 0.2 * n
        th[n, :, :3] = torch.tensor([[math.cos(a), -math.sin(a), 0.05], [math.sin(a), math.cos(a), -0.1], [0.02, 0.1, 1.05]])
        th[n, :, 3] = 0.1 * torch.randn(3, generator=g)
    return th.contiguous()


def inputs(c: Case, device) -> dict:
    """seeded float32 operands of a case"""
    k, g = c.k, gen(c)
    t = {}
    if c.op == "apply":
        N, C = k["N"], k["C"]
        t["x"] = torch.randn((N,) + k["sp"] + (C,), generator=g) * 2 + 0.5
        if k["src"] in ("AB", "AB[n]"):
            t["A"] = torch.randn(N if k["src"] == "AB[n]" else 1, C, generator=g)
            t["B"] = torch.randn(t["A"].shape, generator=g)
        if k["src"].startswith("gn"):
            G = 4
            r = t["x"].double().reshape(N, -1, G, C // G)
            t["stats"] = torch.stack([r.sum((1, 3)), (r * r).sum((1, 3))], -1).contiguous()
            t["gamma"], t["beta"] = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
            if k["src"] == "gn+ada":
                t["ada_w"], t["ada_b"] = torch.rand(N, C, generator=g) + 0.5, torch.randn(N, C, generator=g)
        if k["res"] != "nores":
            t["res"] = torch.randn(t["x"].shape, generator=g)
            if k["res"] == "res+A2B2":
                t["A2"], t["B2"] = torch.randn(C, generator=g), torch.randn(C, generator=g)
    elif c.op == "gn_stats":
        t["x"] = torch.randn((k["N"],) + k["sp"] + (k["C"],), generator=g) * 1.5 - 0.7
    elif c.op == "gn_finalize":
        N, C, G = k["N"], k["C"], k["G"]
        mean, var = torch.randn(N, G, generator=g).double(), torch.rand(N, G, generator=g).double() * 3 + 0.01
        t["count"] = 4096.0
        t["stats"] = torch.stack([mean * 4096, (var + mean * mean) * 4096], -1).contiguous()
        t["gamma"], t["beta"] = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
        if k["ada"]:
            t["ada_w"], t["ada_b"] = torch.rand(N, C, generator=g) + 0.5, torch.randn(N, C, generator=g)
    elif c.op == "gn_head":
        N, C = k["N"], k["C"]
        t["x"] = torch.randn((N,) + k["sp"] + (C,), generator=g) * 1.7 + 0.3
        r = t["x"].double().reshape(N, -1, 32, C // 32)
        t["stats"] = torch.stack([r.sum((1, 3)), (r * r).sum((1, 3))], -1).contiguous()
        t["gamma"], t["beta"] = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
        t["w"], t["bias"] = torch.randn(k["Cout"], C, generator=g) / C ** 0.5, torch.randn(k["Cout"], generator=g)
    elif c.op == "grid_sample3d":
        D, H, W = k["ins"]
        x = torch.randn((k["N"], k["C"], D, H, W), generator=g)
        t["x"] = x if k["layout"] == "ncdhw" else x.permute(0, 2, 3, 4, 1).contiguous()
        if k["coord"] == "theta":
            t["theta"] = gs3_theta(c, g)
        else:
            t["grid"] = gs3_grid(c, g)
    elif c.op in ("upsample_trilinear", "avgpool"):
        t["x"] = torch.randn((k["N"],) + k["sp"] + (k["C"],), generator=g) * 1.3 + 0.4
        if k["add"]:
            t["add"] = torch.randn(out_specs(c)["out"][0], generator=g)
    elif c.op == "linear":
        M, Nn, K = k["M"], k["N"], k["K"]
        t["x"] = torch.randn(max(k["xs"][0] * (M - 1) + k["xs"][1] * (K - 1) + 1, 1), generator=g)
        t["w"] = torch.randn(Nn, K, generator=g) / K ** 0.5
        if k["bias"]:
            t["bias"] = torch.randn(Nn, generator=g)
        if k["add"]:
            t["add"] = torch.randn(out_specs(c)["out"][0], generator=g)
    elif c.op == "conv_direct":
        H, W = k["sp"]
        x = torch.zeros(k["N"], 1, H, W, k["cin"])
        x[..., :3] = torch.rand(k["N"], 1, H, W, 3, generator=g)                     # RGB, padded channels zero
        t["x"] = x
        w = torch.zeros(k["k"], k["k"], k["cin"], k["Cout"])
        w[:, :, :3] = torch.randn(k["k"], k["k"], 3, k["Cout"], generator=g) * 0.1
        t["w"], t["bias"] = w, torch.randn(k["Cout"], generator=g)
    elif c.op == "maxpool2d_3x3s2":
        x = torch.randn(k["N"], 1, k["H"], k["W"], k["C"], generator=g)
        t["x"] = -(x.abs() + 0.25) if k["neg"] else x
    elif c.op == "global_avgpool":
        t["x"] = torch.randn(k["N"], k["S"], k["C"], generator=g) + 1.0
    elif c.op in ("resize_bilinear", "grid_sample2d_affine"):
        t["x"] = torch.rand((k["N"], k["C"]) + k["ins"], generator=g)
        if k["norm"]:
            t["mean"], t["std"] = torch.rand(k["C"], generator=g) * 0.5 + 0.2, torch.rand(k["C"], generator=g) * 0.2 + 0.15
        if c.op == "grid_sample2d_affine":
            th = torch.tensor([[0.7, 0.2, 0.45], [-0.15, 0.8, -0.4]]).repeat(k["N"], 1, 1)
            t["theta"] = (th + 0.05 * torch.randn(th.shape, generator=g)).contiguous()   # maps part of the lattice off the image
    elif c.op in ("split_bf16", "split_f16"):
        x = torch.randn(k["n"], generator=g) * torch.exp2(torch.randint(-12, 10, (k["n"],), generator=g).float())
        x[:4] = torch.tensor([0.0, -0.0, 3.0e-8, 1000.0])
        t["x"] = x
    elif c.op == "stem_pack":
        x = torch.zeros(k["N"], 1, k["H"], k["W"], 4)
        x[..., :3] = (torch.randn(k["N"], 1, k["H"], k["W"], 3, generator=g) * 1.5).clamp(-2.2, 2.7)   # normalised RGB
        t["x"] = x
    elif c.op == "pose_theta":
        t.update(pose_inputs(c, g))
    return {n: (v.to(device) if isinstance(v, torch.Tensor) else v) for n, v in t.items()}


# the clamp's edges (it compares against the fp32 pi), exactly and one fp32 step either side of each, and 0
POSE_EDGES = [-PR.PI32 / 2, PR.PI32, math.nextafter(-PR.PI32 / 2, -4.0), math.nextafter(PR.PI32, 4.0),
              math.nextafter(-PR.PI32 / 2, 0.0), math.nextafter(PR.PI32, 0.0), 0.0]


def _srt(N, g, angles):
    """(N, 9) fp32 (scale 0.6-1.4, yaw pitch roll, translation +-0.5): wider than the head-pose regressor's range"""
    s = 0.6 + 0.8 * torch.rand(N, 3, generator=g, dtype=torch.float64)
    tr = torch.rand(N, 3, generator=g, dtype=torch.float64) - 0.5
    if angles == "inside":
        r = -1.5 + 4.5 * torch.rand(N, 3, generator=g, dtype=torch.float64)
    elif angles == "beyond":
        r = -5.0 + 10.0 * torch.rand(N, 3, generator=g, dtype=torch.float64)
        r[0] = torch.tensor([-2.5, 4.0, -3.0])                           # every axis clamped, on both sides when N > 1
        r[-1] = torch.tensor([4.5, -2.0, 3.7])
    else:
        r = torch.tensor([[POSE_EDGES[(n + 3 * a) % len(POSE_EDGES)] for a in range(3)] for n in range(N)], dtype=torch.float64)
    return torch.cat([s, r, tr], 1).float()


def _sheared_affine(N, g):
    """(N, 4, 4) fp32 rotation . (scale 0.6-1.4 + shear up to 0.15) with translation +-0.5, last row [0, 0, 0, 1]: the polar
    factors of its 3x3 part are not a rotation and a diagonal"""
    th = torch.zeros(N, 4, 4, dtype=torch.float64)
    for n in range(N):
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
        st = torch.diag(0.6 + 0.8 * torch.rand(3, generator=g, dtype=torch.float64))
        st += torch.triu(0.3 * torch.rand(3, 3, generator=g, dtype=torch.float64) - 0.15, 1)
        th[n, :3, :3] = q @ st
        th[n, :3, 3] = torch.rand(3, generator=g, dtype=torch.float64) - 0.5
    th[:, 3, 3] = 1.0
    return th.float()


def pose_inputs(c: Case, g) -> dict:
    """srt or theta_in, the source pose of a mixing case (of the same kind) and the state a carried smoothing case starts from"""
    k, t = c.k, {}
    if k["src"] == "srt":
        t["srt"] = _srt(k["N"], g, k["angles"])
    else:
        t["theta_in"] = _sheared_affine(k["N"], g)
    if k["mix"] != "nomix":
        t["source_theta"] = (torch.from_numpy(PR.srt_theta(_srt(1, g, "inside"))).float() if k["src"] == "srt"
                             else _sheared_affine(1, g))[0].contiguous()
    if "smooth" in k and not k["init"]:
        t["state0"] = torch.from_numpy(PR.srt_theta(_srt(1, g, "inside"))[0, :3]).float().contiguous()
    return t


def out_specs(c: Case) -> dict:
    """{output: (shape, dtype)} of a case; operand planes are (planes, ...shape)"""
    k = c.k
    if c.op == "apply":
        N, (D, H, W), C, up = k["N"], k["sp"], k["C"], k["up"]
        shape = (N, D, H * up, W * up, C)
        o = {"out": (shape, torch.float32)} if "fp32" in k["out"] else {}
        for p in k["out"]:
            if p != "fp32":
                o["planes"] = ((PLANES[p][0],) + shape, PLANES[p][1])
        return o
    if c.op == "gn_stats":
        return {"stats": ((k["N"], k["G"], 2), torch.float64)}
    if c.op == "gn_finalize":
        return {"A": ((k["N"], k["C"]), torch.float32), "B": ((k["N"], k["C"]), torch.float32)}
    if c.op == "gn_head":
        return {"out": ((k["N"], k["Cout"], math.prod(k["sp"])), torch.float32)}
    if c.op == "grid_sample3d":
        N, C, (Do, Ho, Wo) = k["N"], k["C"], k["outs"]
        shape = {"cl": (N, Do, Ho, Wo, C), "hwdc": (N, Ho, Wo, Do, C), "ncdhw": (N, C, Do, Ho, Wo)}[k["out_layout"]]
        o = {"out": (shape, torch.float32)} if k["f32"] else {}
        if k["planes"] != "none":
            o["planes"] = ((PLANES[k["planes"]][0],) + shape, PLANES[k["planes"]][1])
        return o
    if c.op in ("upsample_trilinear", "avgpool"):
        N, (D, H, W), C, f = k["N"], k["sp"], k["C"], k["f"]
        shape = (N, D * f[0], H * f[1], W * f[2], C) if c.op == "upsample_trilinear" else (N, D // f[0], H // f[1], W // f[2], C)
        o = {"out": (shape, torch.float32)}
        if k["stats"]:
            o["stats"] = ((N, 16, 2), torch.float64) if C % 16 == 0 else ((N, 4, 2), torch.float64)
        return o
    if c.op == "linear":
        M, Nn = k["M"], k["N"]
        return {"out": ((k["os"][0] * (M - 1) + k["os"][1] * (Nn - 1) + 1,), torch.float32)}
    if c.op == "conv_direct":
        H, W = k["sp"]
        p, s, kk = kk_pad(c), k["stride"], k["k"]
        o = {"out": ((k["N"], 1, (H + 2 * p - kk) // s + 1, (W + 2 * p - kk) // s + 1, k["Cout"]), torch.float32)}
        if k["stats"]:
            o["stats"] = ((k["N"], k["G"], 2), torch.float64)
        return o
    if c.op == "maxpool2d_3x3s2":
        return {"out": ((k["N"], 1, (k["H"] - 1) // 2 + 1, (k["W"] - 1) // 2 + 1, k["C"]), torch.float32)}
    if c.op == "global_avgpool":
        return {"out": ((k["N"], k["C"]), torch.float32)}
    if c.op in ("resize_bilinear", "grid_sample2d_affine"):
        o = {"out": ((k["N"], 1) + k["outs"] + (k["C_pad"],), torch.float32)}
        if k.get("nchw"):
            o["nchw"] = ((k["N"], k["C"]) + k["outs"], torch.float32)
        return o
    if c.op in ("split_bf16", "split_f16"):
        return {"planes": ((k["planes"], k["n"]), torch.bfloat16 if c.op == "split_bf16" else torch.float16)}
    if c.op == "stem_pack":
        return {"out": ((k["N"], 1, k["H"], k["W"], 32), torch.float16)}
    if c.op == "pose_theta":
        o = {"theta_out": ((k["N"], 4, 4), torch.float32), "theta_warp": ((k["N"], 3, 4), torch.float32)}
        if k["align"]:
            o["align2d"] = ((k["N"], 2, 3), torch.float32)
        if "smooth" in k:
            o["smooth_state"] = ((3, 4), torch.float32)
        return o
    raise KeyError(c.op)


def kk_pad(c: Case) -> int:
    return c.k["k"] // 2


def launch(c: Case, ops, t: dict, o: dict):
    """(entry point, arguments) of the case's C-ABI call on operands `t` and outputs `o` (ops: emoportraits_b200.ops)"""
    from emoportraits_b200 import lib as L

    k, p = c.k, ops._p
    name = "emo_" + c.op
    pl = o.get("planes")
    pp = [p(pl[i]) for i in range(pl.shape[0])] + [None] * (3 - pl.shape[0]) if pl is not None else [None] * 3
    f16 = pl is not None and pl.dtype == torch.float16
    if c.op == "apply":
        gn = None
        if "stats" in t:
            gn = dict(stats=t["stats"], count=t["x"][0].numel() / t["stats"].shape[1], gamma=t["gamma"], beta=t["beta"],
                      ada_w=t.get("ada_w"), ada_b=t.get("ada_b"))
        d, _, _ = ops._apply_desc(p(t["x"]), t["x"].shape, t["x"].device, t.get("A"), t.get("B"), k["act"], t.get("res"), t.get("A2"),
                                  t.get("B2"), k["up"], want_f32=False, want_split=False, per_sample=k["src"] == "AB[n]", gn=gn)
        d.out, (d.out_hi, d.out_lo, d.out_lo2) = p(o.get("out")), pp
        d.plane_fp16, d.plane_scale = (1, F16_SCALE) if f16 else (0, 0.0)
        return name, (C.byref(d), ops._stream())
    if c.op == "gn_stats":
        x = t["x"]
        return name, (p(x), k["N"], x[0].numel() // k["C"], k["C"], k["G"], p(o["stats"]), ops._stream())
    if c.op == "gn_finalize":
        d = L.GnFinalizeDesc(p(t["stats"]), k["N"], k["C"], k["G"], t["count"], 1e-5, p(t["gamma"]), p(t["beta"]),
                             p(t.get("ada_w")), p(t.get("ada_b")), p(o["A"]), p(o["B"]))
        return name, (C.byref(d), ops._stream())
    if c.op == "gn_head":
        x, N, Cc = t["x"], k["N"], k["C"]
        d = L.GnHeadDesc(p(x), N, Cc, x[0].numel() // Cc, p(t["stats"]), 32, x[0].numel() / 32, 1e-5, p(t["gamma"]), p(t["beta"]),
                         p(t["w"]), p(t["bias"]), k["Cout"], k["act"], p(o["out"]))
        return name, (C.byref(d), ops._stream())
    if c.op == "grid_sample3d":
        N, Cc, (Di, Hi, Wi), (Do, Ho, Wo) = k["N"], k["C"], k["ins"], k["outs"]
        os_ = {"ncdhw": (Cc * Do * Ho * Wo, Do * Ho * Wo, Ho * Wo, Wo, 1), "cl": (Do * Ho * Wo * Cc, 1, Ho * Wo * Cc, Wo * Cc, Cc),
               "hwdc": (Do * Ho * Wo * Cc, 1, Cc, Wo * Do * Cc, Do * Cc)}[k["out_layout"]]
        d = L.GridSample3dDesc(p(t["x"]), 1 if k["layout"] == "cl" else 0, N, Cc, Di, Hi, Wi, p(t.get("grid")), p(t.get("theta")),
                               Do, Ho, Wo, p(o.get("out")), pp[0], pp[1], *os_, pp[2], 1 if f16 else 0, F16_SCALE if f16 else 0.0)
        return name, (C.byref(d), ops._stream())
    if c.op in ("upsample_trilinear", "avgpool"):
        x, st = t["x"], o.get("stats")
        d = L.ResampleDesc(p(x), k["N"], *k["sp"], k["C"], *k["f"], p(t.get("add")), p(o["out"]), p(st),
                           st.shape[1] if st is not None else 0)
        return name, (C.byref(d), ops._stream())
    if c.op == "linear":
        d = L.LinearDesc(p(t["x"]), *k["xs"], p(t["w"]), p(t.get("bias")), p(t.get("add")), k["scale"], k["act"], k["M"], k["N"],
                         k["K"], p(o["out"]), *k["os"])
        return name, (C.byref(d), ops._stream())
    if c.op == "conv_direct":
        x, st = t["x"], o.get("stats")
        _, _, Ho, Wo, _ = o["out"].shape
        d = L.ConvDirectDesc(p(x), k["N"], *k["sp"], k["cin"], p(t["w"]), k["Cout"], k["k"], k["k"], k["stride"], kk_pad(c), Ho, Wo,
                             p(t["bias"]), p(o["out"]), p(st), k["G"] if st is not None else 0)
        return name, (C.byref(d), ops._stream())
    if c.op == "maxpool2d_3x3s2":
        return name, (p(t["x"]), k["N"], k["H"], k["W"], k["C"], p(o["out"]), ops._stream())
    if c.op == "global_avgpool":
        return name, (p(t["x"]), k["N"], k["S"], k["C"], p(o["out"]), ops._stream())
    if c.op == "resize_bilinear":
        d = L.ResizeBilinearDesc(p(t["x"]), k["N"], k["C"], *k["ins"], *k["outs"], p(t.get("mean")), p(t.get("std")), p(o["out"]),
                                 k["C_pad"])
        return name, (C.byref(d), ops._stream())
    if c.op == "grid_sample2d_affine":
        d = L.GridSample2dAffineDesc(p(t["x"]), k["N"], k["C"], *k["ins"], p(t["theta"]), *k["outs"], p(t.get("mean")),
                                     p(t.get("std")), p(o["out"]), k["C_pad"], p(o.get("nchw")))
        return name, (C.byref(d), ops._stream())
    if c.op == "split_bf16":
        return name, (p(t["x"]), k["n"], pp[0], pp[1], pp[2], ops._stream())
    if c.op == "split_f16":
        return name, (p(t["x"]), k["n"], C.c_float(F16_SCALE), pp[0], pp[1], ops._stream())
    if c.op == "stem_pack":
        return name, (p(t["x"]), k["N"], k["H"], k["W"], 4, C.c_float(F16_SCALE), p(o["out"]), ops._stream())
    if c.op == "pose_theta":
        st = o.get("smooth_state")
        if st is not None and not k["init"]:
            st.copy_(t["state0"])            # smooth_state is read and written: a carried case starts from the seeded state
        d = ops.pose_desc(k["N"], p(t.get("srt")), p(t.get("source_theta")), p(o["theta_out"]), p(o["theta_warp"]),
                          p(o.get("align2d")), p(t.get("theta_in")), p(st), mix=k["mix"] != "nomix", invert_warp=k["invert"],
                          mix_old=k["mix"] == "mix_old", smooth_init=k.get("init", False), smooth_momentum=k.get("smooth", 0.5))
        return name, (C.byref(d), ops._stream())
    raise KeyError(c.op)


# GroupNorm far from zero mean: the statistics producers accumulate (sum, sum of squares) and every consumer finalises with
# var = q / n - mean^2, whose rounding error grows like (mean / std)^2.  The largest per-group |mean| / std of any GroupNorm
# input of stage 1 at 256^2 and 512^2 (seeded synthetic checkpoint, oracle/frames.py frames) was 2.45 when measured;
# tests/test_op_cases_cpu.py keeps the models under GN_MODEL_RATIO and tests/test_op_cases_gpu.py asserts the 2e-5 bar of
# every producer up to twice that, and at least up to 10: the ratio comes from synthetic weights.  The tightest producer at
# 10 is the convolution epilogue's per-group statistics: 1.2e-5 on an H100, 1.65x under the bar.
GN_MODEL_RATIO = 3.0
GN_ASSERTED_RATIO = max(10.0, 2 * GN_MODEL_RATIO)
