"""GPU replay of every implicit-GEMM convolution the shipped models launch (tests/model_conv_launches.json: stage 1 at 256^2
and 512^2 in exact mode, fast mode and with the fast source pass, stage 2 at 512^2 batch 1 and 1024^2 batch 4 and 16, exact
and fast), at its real shape, against float64.

Each launch is rebuilt from its recorded emo_conv_desc / emo_apply_desc scalars and called through lib.call, so the test runs
exactly the fields the model passed.  Operands are seeded; every output (the convolution's, the post-op's fp32 tensor and
operand planes) and the split-K workspace start as NaN, each followed by a NaN guard region.  Per launch:
  * the live plan equals the recorded one field for field (on 132-SM devices);
  * every output element is written (the fused split-K post kernel writes only the post-op's outputs) and no guard changes;
  * the convolution output is within 1e-5 of max(1, scale) of float64 evaluated on the products the kernel issues: the operand
    planes read back from the device, plane pairs (i, j) with i + j < planes (one plane hi*hi; two hi*hi + hi*lo + lo*hi),
    x out_scale for fp16 planes, then bias, residual (nearest-upsampled with res_shift), activation, post_add;
  * GroupNorm statistics give the float64 per-group mean and mean square;
  * the post-op fp32 output is within 5e-5 of float64 GroupNorm / affine / AdaGN of the reference, [+ res * A2 + B2], activation;
    planes written next to it are its host split bit for bit, planes written alone are within their format's rounding of it;
  * two runs give bit-identical outputs and statistics equal to 1e-13 relative (DESIGN.md section 2.4).
Samples 0 and N - 1 are compared in full at batch 16 (the whole batch is checked for NaN); every sample otherwise."""
import ctypes as C
import math
import time
import zlib

import pytest
import torch
import torch.nn.functional as F

import model_conv_launches as MCL

pytestmark = pytest.mark.gpu
GUARD = 4096
TOL = 1e-5          # convolution: max-abs error / max(1, scale) against the float64 of the issued products
POST_TOL = 5e-5     # post-op: max-abs error / max(1, largest |reference|)
STATS_REPRO = 1e-13
FULL_BATCH = 4      # larger batches compare samples 0 and N - 1 against float64
ROWS = MCL.load()
_WORST_KERNEL, _WORST_CONFIG, _SKIPPED, _T0 = {}, {}, [], []


def _id(i, r):
    d, p = r["conv"], r["post"]
    s = (f"{i:03d}-N{d['N']}-{d['Din']}x{d['Hin']}x{d['Win']}x{d['Cin']}-{d['Cout']}-k{d['kd']}{d['kh']}{d['kw']}s{d['sh']}"
         f"-{_planes_name(d, r['conv_ptrs'])}")
    s += "-up" if d["upconv"] else ""
    s += f"-rs{d['res_shift']}" if d["res_shift"] else ""
    return s + ("-post" if p else "")


def _planes_name(d, ptrs):
    if d["operand_fp16"]:
        return "h2" if "a_lo" in ptrs else "h1"
    return "b3" if "a_lo2" in ptrs else "b2"


# ------------------------------------------------------------------------------------------------------------------
# float64 references on one channels-last sample
# ------------------------------------------------------------------------------------------------------------------
def conv_cl(x, w, stride, pad):
    """x (D, H, W, Cin), w (kd, kh, kw, Cin, Cout) -> (Do, Ho, Wo, Cout): the zero-padded convolution as a sum over taps of
    (shifted x) @ w[tap]"""
    kd, kh, kw = w.shape[:3]
    xp = F.pad(x, (0, 0, pad[2], pad[2], pad[1], pad[1], pad[0], pad[0]))
    Do, Ho, Wo = ((i + 2 * p - k) // s + 1 for i, k, s, p in zip(x.shape[:3], (kd, kh, kw), stride, pad))
    y = x.new_zeros((Do, Ho, Wo, w.shape[-1]))
    for a in range(kd):
        for b in range(kh):
            for c in range(kw):
                y += xp[a:a + stride[0] * (Do - 1) + 1:stride[0], b:b + stride[1] * (Ho - 1) + 1:stride[1],
                        c:c + stride[2] * (Wo - 1) + 1:stride[2]] @ w[a, b, c]
    return y


def upconv_cl(x, wf):
    """sub-pixel form of `nearest x2 -> 3x3 conv (pad 1)`: x (1, H, W, Cin) low resolution, wf (4 phases, 2, 2, Cin, Cout) the
    folded weights (ops.fold_upconv_weight) -> (1, 2H, 2W, Cout)"""
    _, H, W, _ = x.shape
    xp = F.pad(x[0], (0, 0, 1, 1, 1, 1))
    y = x.new_zeros((1, 2 * H, 2 * W, wf.shape[-1]))
    for a in (0, 1):
        for b in (0, 1):
            for ty in (0, 1):
                for tx in (0, 1):
                    y[0, a::2, b::2] += xp[ty + a:ty + a + H, tx + b:tx + b + W] @ wf[2 * a + b, ty, tx]
    return y


def _act(y, act):
    return [lambda t: t, torch.relu, torch.sigmoid, torch.tanh][act](y)


def _host_split(y, n_planes, fp16, scale):
    """the operand planes the device writes for fp32 y (common.cuh split_bf16 / split_bf16x3 / split_f16 / f16_plane)"""
    if fp16:
        ys = (y * scale).clamp(-65000.0, 65000.0)
        hi = ys.half()
        return [hi] if n_planes == 1 else [hi, (ys - hi.float()).half()]
    hi = y.bfloat16()
    r = y - hi.float()
    lo = r.bfloat16()
    return [hi, lo] if n_planes == 2 else [hi, lo, (r - lo.float()).bfloat16()]


# relative rounding of a plane sum: the bar of planes written without an fp32 copy (plus POST_TOL of the scale)
PLANE_BOUND = {(False, 2): 2.0 ** -16, (False, 3): 2.0 ** -24, (True, 2): 2.0 ** -21, (True, 1): 2.0 ** -11}


# ------------------------------------------------------------------------------------------------------------------
# one launch
# ------------------------------------------------------------------------------------------------------------------
def _nan_buf(shape, dtype=torch.float32):
    """(NaN-filled tensor of `shape`, the NaN guard region after it, the whole allocation)"""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf[:n].view(shape), buf[n:], buf


def _estimate_bytes(r):
    """device memory the replay of one launch allocates (operands, outputs, workspace, one sample's float64 reference)"""
    d, p = r["conv"], r["post"]
    np_ = {"h1": 1, "h2": 2, "b2": 2, "b3": 3}[_planes_name(d, r["conv_ptrs"])]
    s_in, s_out = d["Din"] * d["Hin"] * d["Win"] * d["Cin"], d["Dout"] * d["Hout"] * d["Wout"] * d["Cout"]
    b = d["N"] * (s_in * 2 * np_ + s_out * 4 * (1 + ("residual" in r["conv_ptrs"])))
    b += 4 * d["splitk_ws_elems"]
    if p:
        b += d["N"] * s_out * (4 * (("out" in r["post_ptrs"]) + ("res" in r["post_ptrs"])) + 2 * 3)
    b += 8 * (s_in * (np_ + 3) + s_out * 8) + 2 * 4 * s_out * 3   # one sample's float64 reference, two samples' run-1 copies
    return b


@pytest.fixture(scope="module")
def env():
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    _T0.append(time.perf_counter())
    return L, ops


@pytest.mark.parametrize("i", range(len(ROWS)), ids=[_id(i, r) for i, r in enumerate(ROWS)])
def test_model_conv_launch_against_float64(env, i):
    L, ops = env
    r = ROWS[i]
    cid = _id(i, r)
    d, p, cptrs, pptrs = r["conv"], r["post"], set(r["conv_ptrs"]), set(r["post_ptrs"] or ())
    N, Cout = d["N"], d["Cout"]
    need = _estimate_bytes(r)
    if need > 4 << 30:
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        if free < need + (2 << 30):
            _SKIPPED.append((cid, r["configs"], need, free))
            msg = f"[{cid}] needs ~{need / 2 ** 30:.1f} GiB, {free / 2 ** 30:.1f} GiB free on the device"
            print("\n" + msg)
            pytest.skip(msg)

    fmt = _planes_name(d, cptrs)
    planes = {"h1": ops.H1, "h2": ops.H2, "b2": 2, "b3": 3}[fmt]
    fp16 = bool(d["operand_fp16"])
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(MCL.key(r).encode()))
    gc = torch.Generator().manual_seed(zlib.crc32(MCL.key(r).encode()))

    def randn(*shape):
        return torch.randn(shape, generator=g, device="cuda")

    def rand(*shape):
        return torch.rand(shape, generator=g, device="cuda")

    # ---- operands ----
    a = ops.Split.empty((N, d["Din"], d["Hin"], d["Win"], d["Cin"]), "cuda", planes)
    a_planes = [t for t in (a.hi, a.lo, a.lo2) if t is not None]
    for n in range(N):   # one sample at a time: the fp32 activations of a whole 1024^2 batch need not exist at once
        s = ops.split_bf16(randn(1, d["Din"], d["Hin"], d["Win"], d["Cin"]), planes)
        for dst, src in zip(a_planes, (s.hi, s.lo, s.lo2)):
            dst[n].copy_(src[0])
        del s
    taps = (d["kd"], d["kh"], d["kw"])
    if d["upconv"]:
        w = torch.randn((Cout, d["Cin"], 3, 3), generator=gc) / math.sqrt(d["Cin"] * 9)
        pw = ops.pack_upconv_weight(w, device="cuda", planes=planes)
    else:
        w = torch.randn((Cout, d["Cin"]) + taps, generator=gc) / math.sqrt(d["Cin"] * math.prod(taps))
        pw = ops.pack_conv_weight(w, device="cuda", planes=planes)
    assert pw.cout_pad == d["Cout_pad"] and pw.k == taps, (pw.cout_pad, pw.k, d)
    w_planes = [t for t in (pw.hi, pw.lo, pw.lo2) if t is not None]
    assert len(w_planes) == len(a_planes)

    Do, Ho, Wo = d["Dout"], d["Hout"], d["Wout"]
    rs = d["res_shift"]
    t = dict(a_hi=a.hi, a_lo=a.lo, a_lo2=a.lo2, w_hi=pw.hi, w_lo=pw.lo, w_lo2=pw.lo2)
    t["bias"] = randn(Cout) if "bias" in cptrs else None
    t["residual"] = randn(N, Do, Ho >> rs, Wo >> rs, Cout) if "residual" in cptrs else None
    t["post_add"] = randn(Do, Ho, Wo, Cout) if "post_add" in cptrs else None
    t["stats"] = torch.zeros((N, d["G"], 2), dtype=torch.float64, device="cuda") if "stats" in cptrs else None
    oshape = (N, Cout, Do, Ho, Wo) if d["out_nchw"] else (N, Do, Ho, Wo, Cout)
    out, out_guard, out_buf = _nan_buf(oshape)
    t["out"] = out
    ws = ws_guard = ws_buf = None
    if "splitk_ws" in cptrs:
        ws, ws_guard, ws_buf = _nan_buf((d["splitk_ws_elems"],))   # NaN, not zero: the finish reads only what the parts wrote
        t["splitk_ws"] = ws
    assert {k for k, v in t.items() if v is not None} | ({"post"} if p else set()) == cptrs, (sorted(t), sorted(cptrs))
    desc = L.ConvDesc(**d, **{k: v.data_ptr() for k, v in t.items() if v is not None})

    pt, pbufs, pd = {}, [], None
    if p:
        C_ = p["C"]
        assert (p["N"], p["D"], p["H"], p["W"], C_) == (N, Do, Ho, Wo, Cout) and p["up"] == 1
        ab = (N, C_) if p["ab_per_sample"] else (C_,)
        if "A" in pptrs:
            pt["A"], pt["B"] = rand(*ab) + 0.5, randn(*ab) * 0.5
        if "res" in pptrs:
            pt["res"] = randn(N, Do, Ho, Wo, C_)
        if "A2" in pptrs:
            pt["A2"], pt["B2"] = rand(C_) + 0.5, randn(C_) * 0.5
        if "gamma" in pptrs:
            pt["gamma"], pt["beta"] = rand(C_) + 0.5, randn(C_) * 0.5
        if "ada_w" in pptrs:
            pt["ada_w"], pt["ada_b"] = 1.0 + 0.25 * randn(N, C_), 0.5 * randn(N, C_)
        if "stats" in pptrs:
            assert "stats" in cptrs and p["count"] == Do * Ho * Wo * C_ / p["G"], p
            pt["stats"] = t["stats"]
        pshape = (N, Do, Ho, Wo, C_)
        pdt = torch.float16 if p["plane_fp16"] else torch.bfloat16
        for k in ("out", "out_hi", "out_lo", "out_lo2"):
            if k in pptrs:
                o, og, ob = _nan_buf(pshape, torch.float32 if k == "out" else pdt)
                pt[k] = o
                pbufs.append((k, og, ob))
        assert set(pt) == pptrs, (sorted(pt), sorted(pptrs))
        pd = L.ApplyDesc(**p, **{k: v.data_ptr() for k, v in pt.items()})
        desc.post = C.cast(C.pointer(pd), C.c_void_p)

    # ---- plan ----
    lib = L.load()
    info = L.ConvPlanInfo()
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    assert lib.emo_conv_plan(C.byref(desc), sms, C.byref(info)) == 0, lib.emo_last_error().decode()
    plan = {f: getattr(info, f) for f, _ in info._fields_}
    if sms == MCL.SM_COUNT:
        assert plan == r["plan"], (plan, r["plan"])
    else:
        print(f"\n[{cid}] {sms} SMs, not {MCL.SM_COUNT}: plan {plan} not checked")
    kern = L.conv_kernel_name(info.kernel)
    fused_post = L.CONV_FINISH[info.finish] == "post"   # the fused split-K post kernel writes only the post-op outputs

    samples = list(range(N)) if N <= FULL_BATCH else [0, N - 1]

    def run():
        for buf in [out_buf] + ([ws_buf] if ws_buf is not None else []) + [b for _, _, b in pbufs]:
            buf.fill_(float("nan"))
        if t["stats"] is not None:
            t["stats"].zero_()
        L.call("emo_conv_igemm", C.byref(desc), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        keep = {k: torch.stack([v[n] for n in samples]) for k, v in pt.items() if k.startswith("out")}
        if not fused_post:
            keep["conv"] = torch.stack([out[n] for n in samples])
        return keep, (t["stats"].clone() if t["stats"] is not None else None)

    first, st1 = run()
    second, st2 = run()

    # ---- every element written, nothing past the end ----
    for n in range(N):
        if not fused_post:
            assert not torch.isnan(out[n]).any(), f"sample {n}: {int(torch.isnan(out[n]).sum())} output elements never written"
        for k, v in pt.items():
            if k.startswith("out"):
                assert not torch.isnan(v[n]).any(), f"sample {n}: post-op {k} has unwritten elements"
    assert torch.isnan(out_guard).all(), "write past the end of the output tensor"
    if ws_guard is not None:
        assert torch.isnan(ws_guard).all(), "write past the end of the split-K workspace"
    for k, og, _ in pbufs:
        assert torch.isnan(og).all(), f"write past the end of the post-op {k}"

    # ---- reproducibility ----
    for k in first:
        if k == "conv" or st1 is None or torch.equal(st1, st2):
            assert torch.equal(first[k], second[k]), f"{k}: two runs differ"
        else:
            print(f"\n[{cid}] statistics differ in the last bits between the runs; post-op {k} compared to {POST_TOL}")
            a1, a2 = first[k].float(), second[k].float()
            assert (a1 - a2).abs().max().item() <= POST_TOL * max(1.0, a1.abs().max().item()), k
    if st1 is not None:
        rel = ((st1 - st2).abs() / st1.abs().clamp_min(1e-30)).max().item()
        assert rel < STATS_REPRO, rel

    # ---- float64 reference, one sample at a time ----
    n_pl = len(a_planes)
    if d["upconv"]:
        wd = [wp.double().view(4, 2, 2, d["Cout_pad"], d["Cin"]).transpose(3, 4)[..., :Cout] for wp in w_planes]
    else:
        wd = [wp.double().view(taps + (d["Cout_pad"], d["Cin"])).transpose(3, 4)[..., :Cout] for wp in w_planes]
    wsum = [sum(wd[:n_pl - i]) for i in range(n_pl)]   # plane pairs (i, j) with i + j < planes: A_i against W_0 + .. + W_(planes-1-i)
    stride, pad = (d["sd"], d["sh"], d["sw"]), (d["pd"], d["ph"], d["pw"])
    worst = 0.0
    msg = f"\n[{cid}] {kern} ksplit {info.ksplit} grid {info.grid} finish {L.CONV_FINISH[info.finish]}:"
    for si, n in enumerate(samples):
        y = 0
        for i in range(n_pl):
            xn = a_planes[i][n].double()
            y = y + (upconv_cl(xn, wsum[i]) if d["upconv"] else conv_cl(xn, wsum[i], stride, pad))
            del xn
        if fp16:
            y = y * d["out_scale"]
        if t["bias"] is not None:
            y = y + t["bias"].double()
        if t["residual"] is not None:
            res = t["residual"][n].double()
            if rs:
                res = res.repeat_interleave(2, 1).repeat_interleave(2, 2)
            y = y + res
            del res
        scale = y.abs().max().item()
        y = _act(y, d["act"])
        if t["post_add"] is not None:
            y = y + t["post_add"].double()
        scale = max(scale, y.abs().max().item())
        if not fused_post:
            got = second["conv"][si]
            got = got.permute(1, 2, 3, 0) if d["out_nchw"] else got
            e = (got.double() - y).abs().max().item()
            worst = max(worst, e / max(1.0, scale))
            msg += f" n{n} {e:.2e} (scale {scale:.1f})"
            assert e < TOL * max(1.0, scale), (n, e, scale)
        G = d["G"]
        if t["stats"] is not None:
            rg = y.reshape(-1, G, Cout // G)
            cnt = rg.numel() // G
            mean, msq = rg.mean((0, 2)), (rg * rg).mean((0, 2))
            d_mean = (st2[n, :, 0] / cnt - mean).abs().max().item()
            d_msq = ((st2[n, :, 1] / cnt - msq).abs() / msq).max().item()
            msg += f" stats {d_mean:.1e}/{d_msq:.1e}"
            assert d_mean < 1e-6 * max(1.0, scale) and d_msq < 1e-5, (n, d_mean, d_msq)
            del rg
        if p:
            if "stats" in pt:
                rg = y.reshape(-1, G, Cout // G)
                mean = rg.mean((0, 2))
                var = (rg * rg).mean((0, 2)) - mean * mean
                rstd = (var + p["eps"]).rsqrt().repeat_interleave(Cout // G)
                mean = mean.repeat_interleave(Cout // G)
                gam, bet = pt["gamma"].double(), pt["beta"].double()
                if "ada_w" in pt:
                    aw, ab_ = pt["ada_w"][n].double(), pt["ada_b"][n].double()
                    gam, bet = gam * aw, bet * aw + ab_
                A = rstd * gam
                B = bet - mean * A
                del rg
            elif "A" in pt:
                A, B = (pt["A"][n], pt["B"][n]) if p["ab_per_sample"] else (pt["A"], pt["B"])
                A, B = A.double(), B.double()
            else:
                A, B = 1.0, 0.0
            z = y * A + B
            if "res" in pt:
                A2, B2 = (pt["A2"].double(), pt["B2"].double()) if "A2" in pt else (1.0, 0.0)
                z = z + pt["res"][n].double() * A2 + B2
            z = _act(z, p["act"])
            pscale = max(1.0, z.abs().max().item())
            pl = [second[k][si] for k in ("out_hi", "out_lo", "out_lo2") if k in second]
            if "out" in second:
                pe = (second["out"][si].double() - z).abs().max().item()
                msg += f" post {pe:.2e}"
                assert pe < POST_TOL * pscale, (n, pe, pscale)
                for k, (got_pl, want) in enumerate(zip(pl, _host_split(second["out"][si], len(pl), bool(p["plane_fp16"]), p["plane_scale"]))):
                    assert torch.equal(got_pl.view(torch.int16), want.view(torch.int16)), f"post-op plane {k} is not the split of its fp32 output"
            elif pl:
                s = sum(q.double() for q in pl) / (p["plane_scale"] if p["plane_fp16"] else 1.0)
                pe = ((s - z).abs() - PLANE_BOUND[(bool(p["plane_fp16"]), len(pl))] * z.abs()).max().item()
                msg += f" post planes excess {pe:.2e}"
                assert pe < POST_TOL * pscale, (n, pe, pscale)
            del z
        del y
    print(msg)
    if worst > _WORST_KERNEL.get(kern, (0.0, ""))[0]:
        _WORST_KERNEL[kern] = (worst, cid)
    for cfg in r["configs"]:
        if worst > _WORST_CONFIG.get(cfg, (0.0, ""))[0]:
            _WORST_CONFIG[cfg] = (worst, cid)


def test_report_model_conv_launches():
    """(runs after the replay) the largest convolution error / max(1, scale) per kernel instantiation and per configuration,
    the skipped launches and the file's wall time"""
    if not _T0:
        pytest.skip("no launch was replayed")
    print(f"\n[model conv launches] {len(ROWS)} distinct launches, {len(_SKIPPED)} skipped, "
          f"wall time {time.perf_counter() - _T0[0]:.1f} s")
    for k, (rel, cid) in sorted(_WORST_KERNEL.items()):
        print(f"  [largest error / scale] {k:12s} {rel:.2e}  ({cid})")
    for k, (rel, cid) in sorted(_WORST_CONFIG.items()):
        print(f"  [largest error / scale] {k:18s} {rel:.2e}  ({cid})")
    for cid, cfgs, need, free in _SKIPPED:
        print(f"  [skipped] {cid} ({', '.join(cfgs)}): needs ~{need / 2 ** 30:.1f} GiB, {free / 2 ** 30:.1f} GiB free")
