"""GPU replay of every non-convolution launch the shipped models issue (tests/model_op_launches.json: stage 1 at 256^2 and
512^2 in exact mode, fast mode and with the fast source pass, stage 2 at 512^2 batch 1 and 1024^2 batch 4 and 16, exact and
fast) and of every wrapper-boundary launch
(model_op_launches.BOUNDARY), at its real shape, against float64.

Each launch is rebuilt from its recorded scalars and called through lib.call; only the pointers are new.  Inputs are seeded and
shaped like the model's data (image-range white-noise frames, whose pixel-to-pixel steps expose source-coordinate errors at
their largest, uint8 frames, a face crop running off the frame for the 2-D affine sampler, a perturbed identity lattice and
model-sized poses for the 3-D sampler).  Every output and every operand plane starts as NaN, each followed by its own NaN guard region.  Per launch:
  * every output element is written and no guard changes;
  * fp32 outputs are within 2e-5 * max(1, scale) of float64 torch of the same op (test_op_cases_gpu.reference); planes written
    next to an fp32 output are its host split bit for bit, planes written alone are within their format's bound;
  * exact ops match bit for bit: max pooling, the same-size repack, the splits, stem_pack, u8_to_image and image_to_u8;
  * parsing_masks: the masks of every pixel whose two best interpolated logits are more than 1e-5 apart are those of torch's
    fp32 interpolation (the op it restates), and the other pixels are under 1e-3 of the total; against float64, labels
    outside the tie band flip in under MASK_FLIP_BOUND of the pixels;
  * grid_sample2d_affine is held to AFFINE2D_TOL instead of 2e-5: its fp32 source coordinates alone exceed 2e-5 on
    white-noise frames (DESIGN.md section 2, item 5);
  * statistics producers (gn_stats, conv_direct, upsample / avgpool with stats) run on data offset so that the largest
    per-group |mean| / std is op_cases.GN_ASSERTED_RATIO; their statistics match float64, and their output normalised by
    the fused apply matches float64 F.group_norm of it.  An apply that consumes statistics gets them built in float64 from
    its input with the recorded G, count and eps;
  * the pose algebra (regressor-range poses, the source pass's pose as the mixing source) is within the per-entry bars of
    its float64 restatement (tests/pose_reference.py), reported as error / bar;
  * two runs give bit-identical outputs (outputs over 1 GiB are compared by per-sample sums of their bit patterns) and
    statistics equal to 1e-13 relative (DESIGN.md section 2.4).
Samples 0 and N - 1 are compared in full at batch >= 16 (the whole batch is checked for NaN); every sample otherwise.

test_wrappers_issue_only_listed_boundary_launches runs the four wrappers live and checks that each boundary launch they
issue has the class and argument pattern of a BOUNDARY entry."""
import ctypes as C
import math
import time
import zlib

import pytest
import torch
import torch.nn.functional as F

import model_op_launches as MOL
import op_cases as OC
import test_op_cases_gpu as TOG

pytestmark = pytest.mark.gpu
GUARD = 4096
TOL = TOG.TOL
# ops whose fp32 source coordinates alone exceed TOL at the model's shapes (DESIGN.md section 2, item 5)
AFFINE2D_TOL = 1e-4           # grid_sample2d_affine: error / max(1, scale); measured 5.5e-5 at 512 -> 128 on white noise
MASK_FLIP_BOUND = 1e-5        # parsing_masks vs float64: pixels outside the 1e-5 tie band whose label flips; measured 5.3e-6
STATS_REPRO = 1e-13
FULL_BATCH = 15               # batches of 16 and more compare samples 0 and N - 1 against float64
BIG = 1 << 30                 # outputs over 1 GiB: the two runs are compared by per-sample fingerprints
# the pose algebra's launches, then those only the fast source pass issues, joined the table after the others: numbered last,
# in that order, so that every other launch keeps its id
_SRCFAST = {"s1-256-srcfast", "s1-512-srcfast"}
_MODEL = [r for r in MOL.load() if r["op"] != "pose_theta" and not set(r["configs"]) <= _SRCFAST]
ROWS = ([("model", r) for r in _MODEL] + [("boundary", r) for r in MOL.BOUNDARY]
        + [("model", r) for r in MOL.load() if r["op"] == "pose_theta"]
        + [("model", r) for r in MOL.load() if r["op"] != "pose_theta" and set(r["configs"]) <= _SRCFAST])
_WORST, _SKIPPED, _T0 = {}, [], []

DESC = {"apply": "ApplyDesc", "gn_finalize": "GnFinalizeDesc", "gn_head": "GnHeadDesc", "grid_sample3d": "GridSample3dDesc",
        "grid_sample2d_affine": "GridSample2dAffineDesc", "resize_bilinear": "ResizeBilinearDesc", "linear": "LinearDesc",
        "upsample_trilinear": "ResampleDesc", "avgpool": "ResampleDesc", "conv_direct": "ConvDirectDesc", "pose_theta": "PoseDesc"}
SIZE_KEYS = ("N", "D", "H", "W", "C", "S", "n", "Din", "Hin", "Win", "Dout", "Hout", "Wout", "Cout", "M", "K", "fd", "fh", "fw", "up")


def _id(i, kind, r):
    a = r["args"]
    return f"{kind[0]}{i:03d}-{r['op']}-" + "-".join(f"{k}{a[k]}" for k in SIZE_KEYS if k in a and k not in ("fd", "fh", "fw") or
                                                    (k in ("fd", "fh", "fw") and a.get(k, 1) != 1))


# ------------------------------------------------------------------------------------------------------------------
# operands and outputs of one launch
# ------------------------------------------------------------------------------------------------------------------
def _plane_fmt(a, ptrs):
    """operand-plane format of an apply / grid-sampler launch, or None"""
    if "out_hi" not in ptrs:
        return None
    if a["plane_fp16"]:
        return "fp16x2" if "out_lo" in ptrs else "fp16x1"
    return "bf16x3" if "out_lo2" in ptrs else "bf16x2"


def _gs3_layout(a):
    C_, Do, Ho, Wo = a["C"], a["Dout"], a["Hout"], a["Wout"]
    for name, st in (("cl", (Do * Ho * Wo * C_, 1, Ho * Wo * C_, Wo * C_, C_)), ("hwdc", (Do * Ho * Wo * C_, 1, C_, Wo * Do * C_, Do * C_)),
                     ("ncdhw", (C_ * Do * Ho * Wo, Do * Ho * Wo, Ho * Wo, Wo, 1))):
        if st == (a["os_n"], a["os_c"], a["os_d"], a["os_h"], a["os_w"]):
            return name
    raise AssertionError(f"unknown output strides {a}")


def out_specs(op, a, ptrs) -> dict:
    """{output pointer: (shape, dtype)}"""
    f32, u8 = torch.float32, torch.uint8
    if op == "apply":
        shape = (a["N"], a["D"], a["H"] * a["up"], a["W"] * a["up"], a["C"])
        pdt = torch.float16 if a["plane_fp16"] else torch.bfloat16
        return {k: (shape, f32 if k == "out" else pdt) for k in ("out", "out_hi", "out_lo", "out_lo2") if k in ptrs}
    if op == "gn_stats":
        return {"stats": ((a["N"], a["G"], 2), torch.float64)}
    if op == "gn_finalize":
        return {"A": ((a["N"], a["C"]), f32), "B": ((a["N"], a["C"]), f32)}
    if op == "gn_head":
        return {"out": ((a["N"], a["Cout"], a["S"]), f32)}
    if op == "grid_sample3d":
        N, C_, Do, Ho, Wo = a["N"], a["C"], a["Dout"], a["Hout"], a["Wout"]
        shape = {"cl": (N, Do, Ho, Wo, C_), "hwdc": (N, Ho, Wo, Do, C_), "ncdhw": (N, C_, Do, Ho, Wo)}[_gs3_layout(a)]
        pdt = torch.float16 if a["plane_fp16"] else torch.bfloat16
        return {k: (shape, f32 if k == "out" else pdt) for k in ("out", "out_hi", "out_lo", "out_lo2") if k in ptrs}
    if op in ("upsample_trilinear", "avgpool"):
        f = (a["fd"], a["fh"], a["fw"])
        sp = (a["D"], a["H"], a["W"])
        sp = tuple(s * k for s, k in zip(sp, f)) if op == "upsample_trilinear" else tuple(s // k for s, k in zip(sp, f))
        o = {"out": ((a["N"],) + sp + (a["C"],), f32)}
        if "stats" in ptrs:
            o["stats"] = ((a["N"], a["G"], 2), torch.float64)
        return o
    if op == "linear":
        return {"out": ((a["os_m"] * (a["M"] - 1) + a["os_n"] * (a["N"] - 1) + 1,), f32)}
    if op == "conv_direct":
        o = {"out": ((a["N"], 1, a["Hout"], a["Wout"], a["Cout"]), f32)}
        if "stats" in ptrs:
            o["stats"] = ((a["N"], a["G"], 2), torch.float64)
        return o
    if op == "maxpool2d_3x3s2":
        return {"out": ((a["N"], 1, (a["H"] - 1) // 2 + 1, (a["W"] - 1) // 2 + 1, a["C"]), f32)}
    if op == "global_avgpool":
        return {"out": ((a["N"], a["C"]), f32)}
    if op in ("resize_bilinear", "grid_sample2d_affine"):
        o = {"out": ((a["N"], 1, a["Hout"], a["Wout"], a["C_pad"]), f32)}
        if "out_nchw" in ptrs:
            o["out_nchw"] = ((a["N"], a["C"], a["Hout"], a["Wout"]), f32)
        return o
    if op in ("split_bf16", "split_f16"):
        dt = torch.bfloat16 if op == "split_bf16" else torch.float16
        return {k: ((a["n"],), dt) for k in ("hi", "lo", "lo2") if k in ptrs}
    if op == "stem_pack":
        return {"out": ((a["N"], 1, a["H"], a["W"], 32), torch.float16)}
    if op == "u8_to_image":
        return {"out": ((a["N"], a["C"], a["H"], a["W"]), f32)}
    if op == "image_to_u8":
        return {"out": ((a["N"], a["H"], a["W"], a["C"]), u8)}
    if op in ("resize_bicubic", "parsing_prepare", "resize_area"):
        return {"out": ((a["N"], a["C"], a["Hout"], a["Wout"]), f32)}
    if op == "composite":
        return {"out": ((a["N"], a["C"], a["H"], a["W"]), f32)}
    if op == "parsing_masks":
        o = {"out": ((4, a["N"], 1, a["Hout"], a["Wout"]), u8)}
        if "labels" in ptrs:
            o["labels"] = ((a["N"], 1, a["Hout"], a["Wout"]), u8)
        return o
    if op == "pose_theta":
        assert "smooth_state" not in ptrs, "the models do not smooth (the wrapper's smoothing is covered by tests/op_cases.py)"
        shapes = {"theta_out": (a["N"], 4, 4), "theta_warp": (a["N"], 3, 4), "align2d": (a["N"], 2, 3)}
        return {k: (s, f32) for k, s in shapes.items() if k in ptrs}
    raise KeyError(op)


def _lattice_grid(N, Do, Ho, Wo, g):
    """identity lattice plus a perturbation that puts a few percent of the points outside [-1, 1]"""
    zs, ys, xs = (torch.linspace(-1, 1, n, device="cuda") for n in (Do, Ho, Wo))
    w, v, u = torch.meshgrid(zs, ys, xs, indexing="ij")
    base = torch.stack([u, v, w], -1)[None].expand(N, Do, Ho, Wo, 3)
    return (base + 0.04 * torch.randn((N, Do, Ho, Wo, 3), generator=g, device="cuda")).contiguous()


def _pose_theta(N, g):
    """(N, 3, 4) affine of a model-sized pose: rotation up to 30 degrees about a random axis, scale 0.8-1.2, translation +-0.2"""
    th = torch.zeros(N, 3, 4, dtype=torch.float64)
    gc = torch.Generator().manual_seed(int(torch.randint(0, 2 ** 31, (1,), generator=g, device="cuda").item()))
    for n in range(N):
        axis = torch.randn(3, generator=gc, dtype=torch.float64)
        axis /= axis.norm()
        ang = math.radians(30.0) * (2 * torch.rand(1, generator=gc).item() - 1)
        K = torch.tensor([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]], dtype=torch.float64)
        R = torch.eye(3, dtype=torch.float64) + math.sin(ang) * K + (1 - math.cos(ang)) * K @ K
        s = 0.8 + 0.4 * torch.rand(1, generator=gc).item()
        th[n, :, :3] = R * s
        th[n, :, 3] = 0.4 * torch.rand(3, generator=gc, dtype=torch.float64) - 0.2
    return th.float().cuda()


def _regressed_srt(N, g):
    """(N, 9) head-pose regressor output of a face: scale 0.8-1.2, yaw / pitch / roll within +-0.8, translation +-0.2"""
    u = torch.rand(N, 9, generator=g, device="cuda")
    return torch.cat([0.8 + 0.4 * u[:, :3], 1.6 * u[:, 3:6] - 0.8, 0.4 * u[:, 6:] - 0.2], 1).contiguous()


def _image(shape, g, lo=0.0, hi=1.0):
    """an image-range (N, C, H, W) frame of white noise: full-range steps between neighbouring pixels, the steepest edges a
    frame can have, so that an error in a source coordinate shows at its largest"""
    return torch.rand(shape, generator=g, device="cuda").mul_(hi - lo).add_(lo)


def _offset_groups(x, G, r):
    """add to every (sample, group) a mean of r times its standard deviation (x is standard-normal noise)"""
    N, C_ = x.shape[0], x.shape[-1]
    v = x.view(N, -1, G, C_ // G)
    v.add_(r)
    return x


def inputs(op, a, ptrs, g) -> dict:
    """seeded operands of one launch (device tensors), shaped like the model's data"""
    dev = "cuda"

    def randn(*shape, s=1.0, m=0.0):
        return torch.randn(shape, generator=g, device=dev).mul_(s).add_(m)

    def rand(*shape, lo=0.0, hi=1.0):
        return torch.rand(shape, generator=g, device=dev).mul_(hi - lo).add_(lo)

    t = {}
    if op == "apply":
        N, C_ = a["N"], a["C"]
        t["x"] = randn(N, a["D"], a["H"], a["W"], C_, s=2.0, m=0.5)
        if "A" in ptrs:
            t["A"], t["B"] = rand(N if a["ab_per_sample"] else 1, C_, lo=0.5, hi=1.5), randn(N if a["ab_per_sample"] else 1, C_)
        if "stats" in ptrs:
            G = a["G"]
            assert a["count"] == a["D"] * a["H"] * a["W"] * (C_ // G), (a["count"], a)
            st = torch.empty(N, G, 2, dtype=torch.float64, device=dev)
            for n in range(N):
                r = t["x"][n].double().view(-1, G, C_ // G)
                st[n, :, 0], st[n, :, 1] = r.sum((0, 2)), (r * r).sum((0, 2))
            t["stats"] = st
            t["gamma"], t["beta"] = rand(C_, lo=0.5, hi=1.5), randn(C_)
            if "ada_w" in ptrs:
                t["ada_w"], t["ada_b"] = rand(N, C_, lo=0.5, hi=1.5), randn(N, C_)
        if "res" in ptrs:
            t["res"] = randn(*t["x"].shape)
        if "A2" in ptrs:
            t["A2"], t["B2"] = randn(C_), randn(C_)
    elif op == "gn_stats":
        t["x"] = _offset_groups(randn(a["N"], a["S"], a["C"]), a["G"], OC.GN_ASSERTED_RATIO)
    elif op == "gn_finalize":
        N, C_, G, cnt = a["N"], a["C"], a["G"], a["count"]
        mean, var = randn(N, G).double(), rand(N, G, lo=0.01, hi=3.0).double()
        t["stats"] = torch.stack([mean * cnt, (var + mean * mean) * cnt], -1).contiguous()
        t["gamma"], t["beta"] = rand(C_, lo=0.5, hi=1.5), randn(C_)
        if "ada_w" in ptrs:
            t["ada_w"], t["ada_b"] = rand(N, C_, lo=0.5, hi=1.5), randn(N, C_)
    elif op == "gn_head":
        N, C_, S = a["N"], a["C"], a["S"]
        assert a["G"] == 32 and a["count"] == S * C_ // 32, a
        t["x"] = randn(N, 1, 1, S, C_, s=1.7, m=0.3)
        r = t["x"].double().view(N, -1, 32, C_ // 32)
        t["stats"] = torch.stack([r.sum((1, 3)), (r * r).sum((1, 3))], -1).contiguous()
        t["gamma"], t["beta"] = rand(C_, lo=0.5, hi=1.5), randn(C_)
        t["w"], t["bias"] = randn(a["Cout"], C_, s=C_ ** -0.5), randn(a["Cout"])
    elif op == "grid_sample3d":
        N, C_ = a["N"], a["C"]
        shape = (N, a["Din"], a["Hin"], a["Win"], C_) if a["in_layout"] == 1 else (N, C_, a["Din"], a["Hin"], a["Win"])
        t["in_"] = randn(*shape)
        if "theta" in ptrs:
            t["theta"] = _pose_theta(N, g)
        else:
            t["grid"] = _lattice_grid(N, a["Dout"], a["Hout"], a["Wout"], g)
    elif op in ("upsample_trilinear", "avgpool"):
        t["x"] = randn(a["N"], a["D"], a["H"], a["W"], a["C"], s=1.3, m=0.4)
        if "add" in ptrs:
            t["add"] = randn(*out_specs(op, a, ptrs)["out"][0])
    elif op == "linear":
        M, Nn, K = a["M"], a["N"], a["K"]
        t["x"] = randn(a["xs_m"] * (M - 1) + a["xs_k"] * (K - 1) + 1)
        t["w"] = randn(Nn, K, s=K ** -0.5)
        if "bias" in ptrs:
            t["bias"] = randn(Nn)
        if "add" in ptrs:
            t["add"] = randn(*out_specs(op, a, ptrs)["out"][0])
    elif op == "conv_direct":
        N, Cp = a["N"], a["Cin_pad"]
        x = torch.zeros(N, 1, a["Hin"], a["Win"], Cp, device=dev)
        x[..., :3] = _image((N, 3, a["Hin"], a["Win"]), g, lo=-2.0, hi=2.5).permute(0, 2, 3, 1)[:, None]   # normalised RGB
        if "stats" in ptrs:
            x[..., 3] = 1.0     # the padded channel carries the GroupNorm offset through the centre tap (see the replay)
        t["x"] = x
        w = torch.zeros(a["kh"], a["kw"], Cp, a["Cout"], device=dev)
        w[:, :, :3] = randn(a["kh"], a["kw"], 3, a["Cout"], s=(3 * a["kh"] * a["kw"]) ** -0.5)
        t["w"] = w
        if "bias" in ptrs:
            t["bias"] = randn(a["Cout"], s=0.1)
    elif op in ("maxpool2d_3x3s2",):
        t["x"] = randn(a["N"], 1, a["H"], a["W"], a["C"])
    elif op == "global_avgpool":
        t["x"] = randn(a["N"], a["S"], a["C"], m=1.0)
    elif op in ("resize_bilinear", "grid_sample2d_affine"):
        t["in_"] = _image((a["N"], a["C"], a["Hin"], a["Win"]), g)
        if "mean" in ptrs:
            t["mean"], t["std"] = rand(a["C"], lo=0.2, hi=0.7), rand(a["C"], lo=0.15, hi=0.35)
        if op == "grid_sample2d_affine":
            # a face crop that runs off the frame (a face near the edge): part of the lattice samples the zero padding
            th = torch.tensor([[0.9, 0.1, 0.05], [-0.1, 0.9, -0.08]], device=dev).repeat(a["N"], 1, 1)
            t["theta"] = (th + 0.05 * randn(*th.shape)).contiguous()
    elif op in ("split_bf16", "split_f16"):
        t["x"] = randn(a["n"], s=2.0)
    elif op == "stem_pack":
        x = torch.zeros(a["N"], 1, a["H"], a["W"], 4, device=dev)
        x[..., :3] = rand(a["N"], 1, a["H"], a["W"], 3, lo=-2.1, hi=2.6)
        t["x"] = x
    elif op == "u8_to_image":
        t["x"] = torch.randint(0, 256, (a["N"], a["H"], a["W"], a["C"]), generator=g, device=dev, dtype=torch.uint8)
    elif op == "image_to_u8":
        x = _image((a["N"], a["C"], a["H"], a["W"]), g, lo=-0.1, hi=1.1)
        x.view(-1)[:: 9973] = float("nan")          # a NaN pixel becomes 0 (header: emo_image_to_u8)
        t["x"] = x
    elif op in ("resize_bicubic", "parsing_prepare", "resize_area"):
        t["x"] = _image((a["N"], a["C"], a["Hin"], a["Win"]), g)
        if op == "parsing_prepare":
            t["mean"], t["std"] = torch.tensor([0.485, 0.456, 0.406], device=dev), torch.tensor([0.229, 0.224, 0.225], device=dev)
    elif op == "composite":
        N, C_, H, W = a["N"], a["C"], a["H"], a["W"]
        t["img"], t["mask"], t["bg"] = _image((N, C_, H, W), g), _image((N, 1, H, W), g), _image((1, C_, H, W), g)[0]
    elif op == "parsing_masks":
        t["x"] = torch.randn((a["N"], a["K"], a["Hin"], a["Win"]), generator=g, device="cuda")    # white-noise logits
    elif op == "pose_theta":
        import pose_reference as PR

        if "srt" in ptrs:
            t["srt"] = _regressed_srt(a["N"], g)
        if "theta_in" in ptrs:
            t["theta_in"] = torch.from_numpy(PR.srt_theta(_regressed_srt(a["N"], g).cpu())).float().cuda()
        if "source_theta" in ptrs:     # the source pass's pose
            t["source_theta"] = torch.from_numpy(PR.srt_theta(_regressed_srt(1, g).cpu())[0]).float().cuda()
    else:
        raise KeyError(op)
    assert set(t) == set(ptrs) - set(out_specs(op, a, ptrs)), (op, sorted(t), ptrs)
    return t


def _estimate_bytes(op, a, ptrs):
    """device memory one replay holds: operands, outputs, one sample's float64 reference (x 8) and fingerprints"""
    spec = out_specs(op, a, ptrs)
    if op in ("split_bf16", "split_f16"):   # compared in chunks of 2^26 elements
        return 3 * 4 * a["n"] + (4 << 30)
    outs = sum(math.prod(s) * torch.empty(0, dtype=dt).element_size() for s, dt in spec.values())
    ins = {"apply": 4 * a.get("N", 1) * a.get("D", 1) * a.get("H", 1) * a.get("W", 1) * a.get("C", 1) * (1 + ("res" in ptrs)),
           "split_bf16": 4 * a.get("n", 0), "split_f16": 4 * a.get("n", 0)}.get(op, outs)
    per_sample = max(outs, ins) // max(1, a.get("N", 1))
    return outs + ins + 16 * per_sample


# ------------------------------------------------------------------------------------------------------------------
# the call
# ------------------------------------------------------------------------------------------------------------------
def _call(L, op, a, p):
    """launch `op` with the recorded scalars `a` and the pointers `p` ({name: tensor})"""
    name = "emo_" + op
    stream = torch.cuda.current_stream().cuda_stream
    if op in DESC:
        d = getattr(L, DESC[op])(**a, **{k: v.data_ptr() for k, v in p.items()})
        L.call(name, C.byref(d), stream)
        return
    vals = []
    for k in OC.POSITIONAL[name]:
        if k in OC.POSITIONAL_POINTERS:
            vals.append(p[k].data_ptr() if k in p else None)
        elif k == "label_sets":
            vals.append((C.c_uint * 4)(*a[k]))
        else:
            vals.append(a[k])
    L.call(name, *vals, stream)


U8_FILL = 0xA5     # byte outputs and their guards start as this value instead of NaN


def _fill(dtype):
    return U8_FILL if dtype == torch.uint8 else float("nan")


def _alloc(shape, dtype, guard_fill=None):
    """(guard region, output view): the output followed by GUARD elements, all NaN (U8_FILL for bytes); `guard_fill` sets
    another guard value (statistics are atomic sums: an add into a NaN guard would leave it NaN)"""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), _fill(dtype), dtype=dtype, device="cuda")
    if guard_fill is not None:
        buf[n:] = guard_fill
    return buf[n:], buf[:n].view(shape)


def _unwritten(v):
    """elements of v still holding the fill value, counted in chunks (v may hold 2^31 elements)"""
    f = v.reshape(-1)
    cnt = 0
    for c in range(0, f.numel(), 1 << 26):
        p = f[c:c + (1 << 26)]
        cnt += int((p == U8_FILL).sum()) if v.dtype == torch.uint8 else int(torch.isnan(p).sum())
    return cnt


def _bits(t):
    return t if t.dtype == torch.uint8 else TOG._bits(t)


def _fingerprint(t, N):
    """per-sample (sum, position-weighted sum) of the bit patterns of a large output"""
    b = _bits(t).reshape(N, -1)
    out = []
    for n in range(N):
        s = w = 0
        for c in range(0, b.shape[1], 1 << 26):
            v = b[n, c:c + (1 << 26)].long()
            s += int(v.sum())
            w += int((v * torch.arange(c + 1, c + 1 + v.numel(), device=v.device)).sum())
        out.append((s, w))
    return out


def _case(op, a, **kw):
    return OC.Case(op, "", tuple(sorted(kw.items())))


def _sample(t, n, N):
    """operands of sample n (per-sample tensors sliced, shared ones kept)"""
    return {k: (v[n:n + 1] if isinstance(v, torch.Tensor) and v.dim() > 1 and v.shape[0] == N and k not in ("w", "bg") else v)
            for k, v in t.items()}


@pytest.fixture(scope="module")
def env():
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    _T0.append(time.perf_counter())
    return L, ops


def _note(kernel, cfgs, rel, cid):
    for k in [kernel] + [f"{kernel} @ {c}" for c in cfgs]:
        if rel > _WORST.get(k, (-1.0, ""))[0]:
            _WORST[k] = (rel, cid)


@pytest.mark.parametrize("i", range(len(ROWS)), ids=[_id(i, k, r) for i, (k, r) in enumerate(ROWS)])
def test_model_op_launch_against_float64(env, i):
    L, ops = env
    kind, r = ROWS[i]
    cid = _id(i, kind, r)
    op, a, ptrs = r["op"], dict(r["args"]), set(r["ptrs"])
    cfgs = r.get("configs", ["boundary"])
    need = _estimate_bytes(op, a, ptrs)
    if need > 4 << 30:
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        if free < need + (2 << 30):
            _SKIPPED.append((cid, cfgs, need, free))
            msg = f"[{cid}] needs ~{need / 2 ** 30:.1f} GiB, {free / 2 ** 30:.1f} GiB free on the device"
            print("\n" + msg)
            pytest.skip(msg)

    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(MOL.key(r).encode()))
    t = inputs(op, a, ptrs, g)
    spec = out_specs(op, a, ptrs)
    o, guards = {}, {}
    for k, (shape, dt) in spec.items():
        guards[k], o[k] = _alloc(shape, dt, TOG.STATS_GUARD if k == "stats" else None)
    N = 1 if op in ("linear", "split_bf16", "split_f16") else a["N"]
    # byte outputs cannot hold NaN: every sample of them is compared (they are small)
    samples = list(range(N)) if N <= FULL_BATCH or any(dt == torch.uint8 for _, dt in spec.values()) else [0, N - 1]
    stats_out = "stats" in spec

    def run():
        for k, v in o.items():
            v.fill_(0.0 if k == "stats" else _fill(v.dtype))       # statistics accumulate (+=)
        _call(L, op, a, {**t, **o})
        torch.cuda.synchronize()
        keep = {}
        for k, v in o.items():
            batched = v.shape[0] == N and N > 1
            keep[k] = _fingerprint(v, N if batched else 1) if v.numel() * v.element_size() > BIG else v.clone()
        return keep

    # statistics producers: offset the data so that the largest per-group |mean| / std of the output is the asserted ratio
    if stats_out and op != "gn_stats":
        run()
        y, G = o["out"], a["G"]
        off = math.inf
        for n in samples:
            m, s = TOG._group_moments(y[n:n + 1].view(1, -1, y.shape[-1]), G)
            off = min(off, (OC.GN_ASSERTED_RATIO * s - m).min().item())
        if op == "conv_direct":
            t["w"][a["kh"] // 2, a["kw"] // 2, 3] += off       # x[..., 3] == 1 inside the image: every output moves by `off`
        else:
            t["x"] += off            # interpolation and averaging weights sum to one: the output moves by `off`

    first = run()
    second = run()

    # ---- every element written, nothing past the end ----
    for k, v in o.items():
        if k == "stats":
            assert (guards[k] == TOG.STATS_GUARD).all(), "stats: write past the end"
        else:
            assert _unwritten(guards[k]) == guards[k].numel(), f"{k}: write past the end"
        if v.dtype != torch.uint8 and op != "linear":      # linear writes the (m, n) lattice only: checked against float64
            assert _unwritten(v) == 0, f"{k}: {_unwritten(v)} elements never written"

    # ---- reproducibility ----
    for k in first:
        if k == "stats":
            rel = ((first[k] - second[k]).abs() / first[k].abs().clamp_min(1e-30)).max().item()
            assert rel < STATS_REPRO, rel
        elif isinstance(first[k], list):
            assert first[k] == second[k], f"{k}: two runs differ"
        else:
            assert torch.equal(_bits(first[k]), _bits(second[k])), f"{k}: two runs differ"
    del first, second

    # ---- against float64 ----
    msg = f"\n[{cid}] {r['cls']}:"
    worst = _check(op, a, ptrs, t, o, samples, N, ops)
    msg += f" error / {'bar' if op == 'pose_theta' else 'scale'} {worst:.2e}"
    if stats_out:
        worst_gn, ratio = _check_groupnorm(op, a, o, t, samples, ops)
        msg += f"; GroupNorm mean/std {ratio:.1f}: normalised-output error {worst_gn:.2e}"
        _note(f"{op} GroupNorm", cfgs, worst_gn, cid)
    print(msg)
    _note(op, cfgs, worst, cid)


def _cmp(got, want, scale, what, exact=False, tol=TOL):
    e = (got.double() - want).abs().max().item()
    if exact:
        assert torch.equal(got.double(), want), f"{what}: not bit-exact (max diff {e:.2e})"
    assert e < tol * max(1.0, scale), (what, e, scale, tol)
    return e / max(1.0, scale)


def _check(op, a, ptrs, t, o, samples, N, ops):
    """compare samples `samples` of every output with float64; returns the largest error / max(1, scale)"""
    worst = 0.0
    fmt = _plane_fmt(a, ptrs) if op in ("apply", "grid_sample3d") else None
    planes_of = lambda v, n: torch.stack([v[k][n] for k in ("out_hi", "out_lo", "out_lo2") if k in v])   # noqa: E731
    if op in ("split_bf16", "split_f16"):
        fmtp = ("bf16x" if op == "split_bf16" else "fp16x") + str(len([k for k in ("hi", "lo", "lo2") if k in ptrs]))
        x, n = t["x"], a["n"]
        for c in range(0, n, 1 << 26):
            pl = torch.stack([o[k][c:c + (1 << 26)] for k in ("hi", "lo", "lo2") if k in o])
            want = TOG.host_planes(x[c:c + (1 << 26)], fmtp)
            assert torch.equal(TOG._bits(pl), TOG._bits(want)), f"planes [{c}, ...) differ from the host split"
            rel, ab = TOG.PLANE_BOUND[fmtp]
            y = x[c:c + (1 << 26)].double()
            assert ((TOG.reconstruct(pl, fmtp) - y).abs() - rel * y.abs() - ab).max().item() <= 0.0
        return 0.0
    if op == "linear":
        c = _case(op, a, M=a["M"], N=a["N"], K=a["K"], xs=(a["xs_m"], a["xs_k"]), os=(a["os_m"], a["os_n"]), scale=a["scale"],
                  act=a["act"])
        ref, scale = TOG.reference(c, t)
        got, want = o["out"], ref["out"]
        assert torch.equal(torch.isnan(got), torch.isnan(want)), "written positions differ from the (m, n) lattice"
        return _cmp(got[~torch.isnan(want)], want[~torch.isnan(want)], scale, "out")
    if op == "gn_finalize":
        c = _case(op, a)
        ref, scale = TOG.reference(c, dict(t, count=a["count"], eps=a["eps"]))
        return max(_cmp(o["A"], ref["A"], scale, "A"), _cmp(o["B"], ref["B"], scale, "B"))
    if op == "global_avgpool":
        return _cmp(o["out"], t["x"].double().mean(1), t["x"].abs().max().item(), "out")
    if op == "pose_theta":      # every output within its float64 bar (tests/pose_reference.py): error / bar
        import pose_reference as PR

        mix = ("mix_old" if a["mix_old"] else "mix") if a["mix"] else "nomix"
        return max(PR.check_outputs(t, o, mix, bool(a["invert_warp"])).values())
    for n in samples:
        ts = _sample(t, n, N)
        if op == "apply":
            if "stats" in ts:
                ts.update(count=a["count"], eps=a["eps"])
            ref, scale = TOG.reference(_case(op, a, N=1, C=a["C"], act=a["act"], up=a["up"]), ts)
            y = ref["y"]
            if "out" in o:
                worst = max(worst, _cmp(o["out"][n], y[0], scale, f"out[{n}]"))
            if fmt:
                pl = planes_of(o, n)
                if "out" in o:
                    assert torch.equal(TOG._bits(pl), TOG._bits(TOG.host_planes(o["out"][n], fmt))), "planes differ from the split of the fp32 output"
                else:
                    rel, ab = TOG.PLANE_BOUND[fmt]
                    e = ((TOG.reconstruct(pl, fmt) - y[0]).abs() - rel * y[0].abs() - ab).max().item()
                    assert e <= TOL * max(1.0, scale), (fmt, e)
                    worst = max(worst, e / max(1.0, scale))     # planes alone: their excess over the format's rounding
            del ref, y
        elif op == "gn_stats":
            ref, _ = TOG.reference(_case(op, a, N=1, C=a["C"], G=a["G"]), ts)
            worst = max(worst, _stats_err(o["stats"][n:n + 1], ref["stats"], ref["abs"]))
        elif op == "gn_head":
            ts["eps"] = a["eps"]
            ref, scale = TOG.reference(_case(op, a, N=1, act=a["act_out"]), ts)
            worst = max(worst, _cmp(o["out"][n], ref["out"][0], scale, "out"))
        elif op == "grid_sample3d":
            ts["x"] = ts.pop("in_")
            layout = "cl" if a["in_layout"] == 1 else "ncdhw"
            ref, scale = TOG.reference(_case(op, a, layout=layout, out_layout=_gs3_layout(a), outs=(a["Dout"], a["Hout"], a["Wout"])), ts)
            y = ref["y"][0]
            if "out" in o:
                worst = max(worst, _cmp(o["out"][n], y, scale, "out"))
            if fmt:
                pl = planes_of(o, n)
                if "out" in o:
                    assert torch.equal(TOG._bits(pl), TOG._bits(TOG.host_planes(o["out"][n], fmt)))
                else:
                    rel, ab = TOG.PLANE_BOUND[fmt]
                    e = ((TOG.reconstruct(pl, fmt) - y).abs() - rel * y.abs() - ab).max().item()
                    assert e <= TOL * max(1.0, scale), (fmt, e)
                    worst = max(worst, e / max(1.0, scale))
        elif op in ("upsample_trilinear", "avgpool"):
            f = (a["fd"], a["fh"], a["fw"])
            ref, scale = TOG.reference(_case(op, a, f=f), ts)
            worst = max(worst, _cmp(o["out"][n], ref["out"][0], scale, "out", exact=f == (1, 1, 1) and "add" not in ts))
            if "stats" in o:
                worst = max(worst, _producer_stats(o, n, a["G"]))
        elif op == "conv_direct":
            assert a["kh"] == a["kw"] and a["pad"] == a["kh"] // 2, a
            if "bias" not in ts:
                ts["bias"] = torch.zeros(a["Cout"], device="cuda")
            ref, scale = TOG.reference(_case(op, a, stride=a["stride"], k=a["kh"]), ts)
            worst = max(worst, _cmp(o["out"][n], ref["out"][0], scale, "out"))
            if "stats" in o:
                worst = max(worst, _producer_stats(o, n, a["G"]))
        elif op == "maxpool2d_3x3s2":
            ref, _ = TOG.reference(_case(op, a), ts)
            _cmp(o["out"][n], ref["out"][0].double(), 1.0, "out", exact=True)
        elif op in ("resize_bilinear", "grid_sample2d_affine"):
            ts["x"] = ts.pop("in_")
            c = _case(op, a, N=1, C=a["C"], outs=(a["Hout"], a["Wout"]), C_pad=a["C_pad"])
            ref, scale = TOG.reference(c, ts)
            same = op == "resize_bilinear" and (a["Hin"], a["Win"]) == (a["Hout"], a["Wout"]) and "mean" not in ts
            tol = AFFINE2D_TOL if op == "grid_sample2d_affine" else TOL
            worst = max(worst, _cmp(o["out"][n], ref["out"][0], scale, "out", exact=same, tol=tol))
            assert (o["out"][n][..., a["C"]:] == 0).all(), "padding channels not zero"
            if "out_nchw" in o:
                worst = max(worst, _cmp(o["out_nchw"][n], ref["nchw"][0], scale, "out_nchw", tol=tol))
        elif op == "stem_pack":
            import test_fast_stage2_gpu as TS

            want = TS._stem_im2col(ts["x"], a["scale"])
            assert torch.equal(o["out"][n:n + 1].view(torch.int16), want.view(torch.int16)), f"sample {n}: differs from the host im2col"
        elif op == "u8_to_image":
            want = (ts["x"].double() / 255).float().permute(0, 3, 1, 2)
            assert torch.equal(o["out"][n:n + 1], want), f"sample {n}: not u / 255"
        elif op == "image_to_u8":
            want = (torch.nan_to_num(ts["x"], nan=0.0).clamp(0, 1) * 255).to(torch.uint8).permute(0, 2, 3, 1)
            assert torch.equal(o["out"][n:n + 1], want), f"sample {n}: not trunc(clamp(x, 0, 1) * 255)"
        elif op in ("resize_bicubic", "parsing_prepare", "resize_area"):
            x = ts["x"].double()
            size = (a["Hout"], a["Wout"])
            if op == "resize_bicubic":
                y = F.interpolate(x, size=size, mode="bicubic", align_corners=False)
            elif op == "resize_area":
                y = F.interpolate(x * a["scale"] + a["shift"], size=size, mode="area")
            else:
                x = (x - ts["mean"].double()[:, None, None]) / ts["std"].double()[:, None, None]
                y = x if size == (a["Hin"], a["Win"]) else F.interpolate(x, size=size, mode="bilinear", align_corners=False)
            worst = max(worst, _cmp(o["out"][n], y[0], max(x.abs().max().item(), y.abs().max().item()), "out"))
        elif op == "composite":
            m = ts["mask"].double()
            m = torch.where(m > C.c_float(a["threshold"]).value, m, torch.zeros_like(m)) ** 8
            y = m * ts["img"].double() + (1 - m) * t["bg"].double()
            worst = max(worst, _cmp(o["out"][n], y[0], 1.0, "out"))
        elif op == "parsing_masks":
            # the kernel restates F.interpolate on fp32 logits (face_parcing.py), fp32 source coordinates included: against
            # torch's fp32 interpolation every label outside the 1e-5 tie band is equal (as tests/test_masks.py checks);
            # against float64 coordinates a few flip where the ratio (512 / 1080) is not exact in fp32: MASK_FLIP_BOUND
            flips = 0.0
            for up in (F.interpolate(ts["x"].cpu(), size=(a["Hout"], a["Wout"]), mode="bilinear", align_corners=False).cuda(),
                       F.interpolate(ts["x"].double(), size=(a["Hout"], a["Wout"]), mode="bilinear", align_corners=False)):
                lab = up.argmax(1, keepdim=True)
                top2 = up.topk(2, dim=1).values
                safe = (top2[:, :1] - top2[:, 1:2]) > 1e-5
                assert (~safe).float().mean().item() < 1e-3
                bad = torch.zeros_like(safe)
                for s, bits in enumerate(a["label_sets"]):
                    want = ((torch.tensor(bits, device=lab.device) >> lab) & 1).to(torch.uint8)
                    bad |= (o["out"][s, n:n + 1] != want) & safe
                frac = bad.float().mean().item()
                if up.dtype == torch.float32:
                    assert not bad.any(), f"sample {n}: {int(bad.sum())} masks differ from torch's fp32 interpolation"
                else:
                    assert frac < MASK_FLIP_BOUND, f"sample {n}: {int(bad.sum())} labels ({frac:.2e}) flip against float64"
                    flips = max(flips, frac)
                del up, top2
            worst = max(worst, flips)
        else:
            raise KeyError(op)
    return worst


def _stats_err(st, want, mag):
    es = ((st[..., 0] - want[..., 0]).abs() / mag).max().item()
    eq = ((st[..., 1] - want[..., 1]).abs() / want[..., 1]).max().item()
    assert es < 2e-6 and eq < 2e-6, (es, eq)
    return max(es, eq)


def _producer_stats(o, n, G):
    """the producer's statistics against float64 of its own output (sample n)"""
    y = o["out"][n:n + 1].double()
    rr = y.reshape(1, -1, G, y.shape[-1] // G)
    return _stats_err(o["stats"][n:n + 1], torch.stack([rr.sum((1, 3)), (rr * rr).sum((1, 3))], -1), rr.abs().sum((1, 3)))


def _check_groupnorm(op, a, o, t, samples, ops):
    """(largest error, achieved |mean| / std) of the producer's output normalised by the fused apply with its statistics,
    against float64 F.group_norm of that output"""
    G = a["G"]
    y_all = t["x"] if op == "gn_stats" else o["out"]
    worst, ratio = 0.0, 0.0
    for n in samples:
        y = y_all[n:n + 1]
        y = y.view(1, 1, 1, -1, y.shape[-1])
        Cc = y.shape[-1]
        ones, zeros = torch.ones(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
        count = y[0].numel() / G
        if op != "gn_stats":
            assert count * G == y[0].numel()
        z = ops.apply(y, gn=dict(stats=o["stats"][n:n + 1], count=count, gamma=ones, beta=zeros), want_f32=True, want_split=False)
        torch.cuda.synchronize()
        ref = TOG._cl(F.group_norm(TOG._ncdhw(y.double()), G, eps=1e-5))
        m, s = TOG._group_moments(y, G)
        ratio = max(ratio, (m.abs() / s).max().item())
        e = (z.double() - ref).abs().max().item()
        assert e < TOL, (n, e)
        worst = max(worst, e)
        del z, ref
    assert ratio > 0.9 * OC.GN_ASSERTED_RATIO, ratio
    return worst, ratio


def test_report_model_op_launches():
    """(runs after the replay) the largest error / max(1, scale) per kernel and per kernel and configuration, the skipped
    launches and the file's wall time"""
    if not _T0:
        pytest.skip("no launch was replayed")
    print(f"\n[model op launches] {len(ROWS)} launches, {len(_SKIPPED)} skipped, wall time {time.perf_counter() - _T0[0]:.1f} s")
    for k, (rel, cid) in sorted(_WORST.items()):
        print(f"  [largest error / scale] {k:48s} {rel:.2e}  ({cid})")
    for cid, cfgs, need, free in _SKIPPED:
        print(f"  [skipped] {cid} ({', '.join(cfgs)}): needs ~{need / 2 ** 30:.1f} GiB, {free / 2 ** 30:.1f} GiB free")
    total = torch.cuda.get_device_properties(torch.cuda.current_device()).total_memory
    assert not (_SKIPPED and total >= 80e9), f"{len(_SKIPPED)} launches skipped on a {total / 1e9:.0f} GB device"


def test_wrappers_issue_only_listed_boundary_launches(tmp_path):
    """the four wrappers run live: stage 1 at 256^2 with a 640x480 source and a list of 4 drivers, stage 2 at 512^2 batch 2,
    the video loop with a background and a matte, and the mask helpers with the stand-in networks.  Every boundary launch
    they issue has the class and argument pattern (the record without its sizes) of a BOUNDARY entry, and every boundary
    entry point is reached."""
    import pathlib

    from emoportraits_b200 import lib as L
    from emoportraits_b200 import video
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper
    from emoportraits_b200.masks import FaceParsing, modnet_get_mask
    from emoportraits_b200.stage2 import InferenceWrapper as Stage2Wrapper
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2
    from oracle import frames as FR
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    gold = pathlib.Path(__file__).parent / "golden"
    boundary_ops = {r["op"] for r in MOL.BOUNDARY}
    listed = {MOL.pattern(r) for r in MOL.BOUNDARY}
    seen = []
    launch = L.call

    def call(name, *args):
        if name[4:] in boundary_ops:
            seen.append(MOL.launch_record(name, args))
        return launch(name, *args)

    size = 256
    cfg = shipped_config(size)
    w1 = InferenceWrapper(experiment_name="x", project_dir=str(tmp_path), args_path=gold / f"args_{size}.txt",
                          state_dict=synthetic_state_dict(cfg, 0), head_pose_state_dict=synthetic_head_pose_state_dict(0),
                          print_params=False)
    cfg2 = Stage2Config(output_size=512)
    ckpt = tmp_path / "logs_s2" / "exp" / "checkpoints"
    ckpt.mkdir(parents=True)
    (tmp_path / "logs_s2" / "exp" / "args.txt").write_text((gold / "args_s2_512.txt").read_text())
    torch.save(synthetic_state_dict_s2(cfg2, 0), ckpt / "m.pth")
    w2 = Stage2Wrapper(experiment_name="exp", model_file_name="m.pth", project_dir=str(tmp_path))
    mp = pytest.MonkeyPatch()
    mp.setattr(L, "call", call)
    try:
        w1.forward(FR.pil(size, 41, "smooth").resize((640, 480)), None, crop=False)
        w1.forward(None, [FR.pil(size, 50 + i, "smooth") for i in range(4)], crop=False)
        w2.forward(torch.rand(2, 3, 512, 512, device="cuda"))
        bg = torch.rand(3, size, size)
        video.drive_image_with_video(w1, FR.pil(size, 41, "smooth"), [FR.pil(size, 60 + i, "smooth") for i in range(3)], bg=bg,
                                     mask_fn=lambda img: torch.rand(img.shape[0], 1, size, size, device="cuda"), chunk=2)
        FaceParsing(None, device="cuda", net=StubBiSeNet().cuda()).forward(torch.rand(1, 3, 512, 512, device="cuda"))
        modnet_get_mask(StubMODNet().cuda(), torch.rand(1, 3, 300, 400, device="cuda"))
        torch.cuda.synchronize()
    finally:
        mp.undo()
    unlisted = [r for r in seen if MOL.pattern(r) not in listed]
    print(f"\n[wrapper boundary] {len(seen)} launches, {len({MOL.key(r) for r in seen})} distinct, {len(unlisted)} unlisted")
    assert not unlisted, unlisted
    assert {r["op"] for r in seen} == boundary_ops, sorted(boundary_ops - {r["op"] for r in seen})
