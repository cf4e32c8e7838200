"""Tensor-in / tensor-out wrappers over the C-ABI (PyTorch is only the owner of device memory and streams).

Layout vocabulary
  "cl"    channels-last activation, fp32, shape (N, D, H, W, C) (D == 1 for 2-D maps)
  Split   the same tensor as two bf16 planes (hi, lo) — the tensor-core operand format
  NCDHW   torch-contiguous layout of the reference (only at the API boundary)
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from dataclasses import dataclass
from typing import Optional

import torch

from . import lib as L
from .lib import ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH  # noqa: F401


def _stream() -> int:
    if L.DRY_RUN:
        return 0
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    assert t.is_cuda or L.DRY_RUN, "emoportraits_b200 ops need CUDA tensors (there is no CPU path)"
    return t.data_ptr()


def _chk(t: torch.Tensor, dtype=torch.float32):
    assert (t.is_cuda or L.DRY_RUN) and t.dtype == dtype and t.is_contiguous(), (t.device, t.dtype, t.is_contiguous())
    return t


# fp16 two-plane operand mode ("h2"): planes hold (value * power of two) so that both fp16 planes stay in the normal range;
# the convolution undoes the two scales on its fp32 sums (emo_conv_desc.operand_fp16 / out_scale).  ~2^-22 per operand:
# fp32-faithful like three bf16 planes, at three MMAs per product instead of six (tools/split_precision_emulation.py).
H2 = "h2"
F16_ACT_SCALE = 16.0    # activations: post-GroupNorm / ReLU values are O(1)
F16_W_SCALE = 256.0     # spectral-norm / weight-standardised weights are O(0.01 .. 1)
# fp16 one-plane operand mode ("h1"): ONE fp16 plane of (value * the same power of two as "h2"), one MMA per product instead of
# three, ~2^-11 relative per operand.  Stage 1's decoder, its source-volume networks (local encoder, volume blocks, 3-D U-Net) and
# stage 2 only, in their fast modes (DESIGN.md section 2): the embedding / warp networks feed the sampler, which amplifies their
# errors ~100x (tools/decoder_precision_emulation.py gives the bounds).
H1 = "h1"


# MMAs per accumulation chunk (the tensor core accumulates with truncation: DESIGN.md section 2).  bf16 two-plane operands
# (decoder, stage 2): 96 - measured round 2 with tools/conv_layer_bench.py: the frame's conv shapes take 2.29 ms at 48, 2.20 ms
# at 96, 2.17 ms at 192, 2.16 ms unchunked; parity of the decoder stage is unchanged at 96 (tests/test_stage_parity_gpu.py).
# fp16 two-plane operands (the fp32-faithful networks) stay at 24: at 48 the frame is 1.5 % faster (285.7 -> 290.1 frames/s) but the
# truncation bias shows - stage errors of the embedders / warp generator grow 1.5-2x (expression embedding 5e-6 -> 1.2e-5) and one
# end-to-end tap leaves its bound; bf16 three-plane operands keep the kernel default 24 as well.
ACC_CHUNK_BF16 = 96
ACC_CHUNK_F16 = 24


def _nplanes(planes) -> int:
    return 2 if planes == H2 else 1 if planes == H1 else int(planes)


@dataclass
class Split:
    """operand planes of a channels-last activation (N, D, H, W, C): bf16 (hi, lo) — or (hi, lo, lo2) in the fp32-faithful
    three-plane mode used by the numerically sensitive networks — or, with f16 = True, fp16 (hi, lo) of value * scale, or
    fp16 hi alone (lo None: the one-plane mode H1)."""
    hi: torch.Tensor
    lo: Optional[torch.Tensor]
    lo2: Optional[torch.Tensor] = None
    f16: bool = False
    scale: float = 1.0

    @property
    def shape(self):
        return self.hi.shape

    @property
    def planes(self) -> int:
        return 3 if self.lo2 is not None else 2 if self.lo is not None else 1

    @staticmethod
    def empty(shape, device, planes=2) -> "Split":
        if planes == H1:
            return Split(torch.empty(tuple(shape), dtype=torch.float16, device=device), None, None, True, F16_ACT_SCALE)
        if planes == H2:
            buf = torch.empty((2,) + tuple(shape), dtype=torch.float16, device=device)
            return Split(buf[0], buf[1], None, True, F16_ACT_SCALE)
        buf = torch.empty((planes,) + tuple(shape), dtype=torch.bfloat16, device=device)
        return Split(buf[0], buf[1], buf[2] if planes == 3 else None)

    def view(self, *shape) -> "Split":
        return Split(self.hi.view(*shape), self.lo.view(*shape) if self.lo is not None else None,
                     self.lo2.view(*shape) if self.lo2 is not None else None, self.f16, self.scale)

    def float(self) -> torch.Tensor:
        f = self.hi.float() + self.lo.float() if self.lo is not None else self.hi.float()
        f = f + self.lo2.float() if self.lo2 is not None else f
        return f / self.scale if self.f16 else f


@dataclass
class PackedConvWeight:
    """Conv weight in the kernel-native layout: bf16 planes [taps][Cout_pad][Cin] (taps = kd*kh*kw); fp16 planes of
    weight * scale with f16 (lo None: the one-plane mode H1)."""
    hi: torch.Tensor
    lo: Optional[torch.Tensor]
    cout: int
    cout_pad: int
    cin: int
    k: tuple  # (kd, kh, kw)
    lo2: Optional[torch.Tensor] = None
    acc_chunk: int = 0  # MMAs per accumulation chunk (0 = kernel default: 16 with one plane, 48 with two, 24 with three)
    f16: bool = False   # fp16 planes of weight * scale (the "h2" / "h1" operand modes)
    scale: float = 1.0


def split_host(w: torch.Tensor, planes=2):
    """fp32 -> bf16 planes (or, planes == "h2" / "h1", two / one fp16 planes of w * F16_W_SCALE) with torch ops (load-time
    weight preparation only)."""
    if planes in (H2, H1):
        assert float(w.abs().max()) * F16_W_SCALE < 6.0e4, "weight too large for the fp16 plane scale"
        ws = w * F16_W_SCALE
        hi = ws.to(torch.float16)
        return (hi,) if planes == H1 else (hi, (ws - hi.float()).to(torch.float16))
    hi = w.to(torch.bfloat16)
    r = w - hi.float()
    lo = r.to(torch.bfloat16)
    if planes == 2:
        return hi, lo
    lo2 = (r - lo.float()).to(torch.bfloat16)
    return hi, lo, lo2


def pack_conv_weight(w: torch.Tensor, device=None, in_perm: Optional[torch.Tensor] = None, planes=2) -> PackedConvWeight:
    """OIHW / OIDHW fp32 (already SN/WS-folded) -> PackedConvWeight. `in_perm` optionally re-orders input channels."""
    w = w.detach().float()
    if w.dim() == 4:
        w = w[:, :, None]
    co, ci, kd, kh, kw = w.shape
    if in_perm is not None:
        w = w[:, in_perm]
    co_pad = ((co + 15) // 16) * 16
    wp = torch.zeros(kd * kh * kw, co_pad, ci, dtype=torch.float32)
    wp[:, :co] = w.permute(2, 3, 4, 0, 1).reshape(kd * kh * kw, co, ci).cpu()
    pl = split_host(wp, planes)
    dev = device or "cuda"
    if planes == H1:
        return PackedConvWeight(pl[0].contiguous().to(dev), None, co, co_pad, ci, (kd, kh, kw), None, 0, True, F16_W_SCALE)
    if planes == H2:
        return PackedConvWeight(pl[0].contiguous().to(dev), pl[1].contiguous().to(dev), co, co_pad, ci, (kd, kh, kw), None, ACC_CHUNK_F16,
                                True, F16_W_SCALE)
    return PackedConvWeight(pl[0].contiguous().to(dev), pl[1].contiguous().to(dev), co, co_pad, ci, (kd, kh, kw),
                            pl[2].contiguous().to(dev) if planes == 3 else None, ACC_CHUNK_BF16 if planes == 2 else 0)


def fold_upconv_weight(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, 3, 3) weights of `nearest x2 -> 3x3 conv (pad 1)` -> (4 phases, 2, 2, Cout, Cin) weights of the four
    2x2 convolutions over the LOW-resolution map that compute the same thing (sub-pixel form).  Output pixel
    (2i + a, 2j + b) reads upsampled rows 2i+a-1 .. 2i+a+1, i.e. low-res rows {i-1, i, i} for a = 0 and {i, i, i+1} for
    a = 1: row taps {w0, w1 + w2} at offsets {-1, 0} (a = 0) and {w0 + w1, w2} at offsets {0, +1} (a = 1); columns alike.
    Zero padding of the upsampled map coincides with zero padding of the low-res map.  phase = 2a + b, taps (ty, tx)."""
    assert w.dim() == 4 and tuple(w.shape[2:]) == (3, 3), w.shape
    w = w.detach().float()
    rows = [torch.stack([w[:, :, 0], w[:, :, 1] + w[:, :, 2]], 2), torch.stack([w[:, :, 0] + w[:, :, 1], w[:, :, 2]], 2)]  # (Co,Ci,2,3) per a
    out = []
    for a in (0, 1):
        r = rows[a]
        for b in (0, 1):
            c = torch.stack([r[..., 0], r[..., 1] + r[..., 2]], 3) if b == 0 else torch.stack([r[..., 0] + r[..., 1], r[..., 2]], 3)
            out.append(c.permute(2, 3, 0, 1))                                  # (ty, tx, Co, Ci)
    return torch.stack(out)                                                    # (4, 2, 2, Co, Ci)


def fold_poolconv_weight(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, 3, 3) weights of `3x3 conv (pad 1) -> 2x2 average pool` -> (Cout, Cin, 4, 4) weights of the ONE
    4x4 stride-2 pad-1 convolution that computes the same thing:
        avgpool2(conv3(x))[i, j] = 1/4 sum_{a,b in {0,1}} sum_{p,q} w[p, q] x[2i+a+p-1, 2j+b+q-1]
                                 = sum_{u,v in 0..3} w4[u, v] x[2i+u-1, 2j+v-1],   w4[u, v] = 1/4 sum_{a,b} w[u-a, v-b].
    16 taps per pooled output instead of 4 x 9, and the full-resolution conv output never exists.  The conv bias passes
    through the pool unchanged."""
    assert w.dim() == 4 and tuple(w.shape[2:]) == (3, 3), w.shape
    w = w.detach().float()
    w4 = torch.zeros(w.shape[0], w.shape[1], 4, 4, dtype=torch.float32)
    for a in (0, 1):
        for b in (0, 1):
            w4[:, :, a:a + 3, b:b + 3] += w
    return 0.25 * w4


def pack_upconv_weight(w: torch.Tensor, device=None, planes=2) -> PackedConvWeight:
    """OIHW 3x3 fp32 (already SN/WS-folded) -> phase-folded PackedConvWeight [16 = phase*4 + ty*2 + tx][Cout][Cin] for
    conv_igemm(..., upconv=True).  Cout must be a multiple of 32 (no padding rows; pair-mode N tiles).  planes: 2 (bf16) or H1."""
    assert planes in (2, H1), "the sub-pixel convolution runs with two bf16 planes or one fp16 plane"
    co, ci = w.shape[:2]
    assert co % 32 == 0 and ci % 64 == 0, (co, ci)
    wp = fold_upconv_weight(w).reshape(16, co, ci).contiguous()
    dev = device or "cuda"
    if planes == H1:
        (hi,) = split_host(wp, H1)
        return PackedConvWeight(hi.contiguous().to(dev), None, co, co, ci, (1, 3, 3), None, 0, True, F16_W_SCALE)
    hi, lo = split_host(wp, 2)
    return PackedConvWeight(hi.contiguous().to(dev), lo.contiguous().to(dev), co, co, ci, (1, 3, 3), None, ACC_CHUNK_BF16)


# ------------------------------------------------------------------------------------------------
# grid_sample
# ------------------------------------------------------------------------------------------------
def grid_sample3d(inp: torch.Tensor, grid: Optional[torch.Tensor] = None, theta: Optional[torch.Tensor] = None,
                  out_size=None, in_layout: str = "ncdhw", out_layout: Optional[str] = None, want_f32: bool = True,
                  want_split: bool = False, planes=2):
    """Trilinear, zeros padding, align_corners=False (va.py:261-265).

    in_layout  'ncdhw' (N,C,D,H,W)  or 'cl' (N,D,H,W,C)
    out_layout 'ncdhw' | 'cl' | 'hwdc' ((N,H,W,D,C): the decoder's flattened-2D layout); default = in_layout
    grid (N,Do,Ho,Wo,3) xyz, or theta (N,3,4) with out_size=(Do,Ho,Wo) for the fused affine lattice.
    want_split: also the operand planes of the output (planes 2 / 3 bf16, or H1: one fp16 plane of y * F16_ACT_SCALE).
    """
    assert planes in (2, 3, H1), "grid_sample3d writes two or three bf16 planes or one fp16 plane"
    _chk(inp)
    if in_layout == "ncdhw":
        N, Cc, Di, Hi, Wi = inp.shape
    else:
        N, Di, Hi, Wi, Cc = inp.shape
    if grid is not None:
        _chk(grid)
        assert grid.shape[0] == N and grid.shape[-1] == 3
        Do, Ho, Wo = grid.shape[1:4]
    else:
        _chk(theta)
        assert theta.shape == (N, 3, 4) and out_size is not None
        Do, Ho, Wo = out_size
    out_layout = out_layout or in_layout
    if out_layout == "ncdhw":
        shape = (N, Cc, Do, Ho, Wo)
        os_ = dict(n=Cc * Do * Ho * Wo, c=Do * Ho * Wo, d=Ho * Wo, h=Wo, w=1)
    elif out_layout == "cl":
        shape = (N, Do, Ho, Wo, Cc)
        os_ = dict(n=Do * Ho * Wo * Cc, c=1, d=Ho * Wo * Cc, h=Wo * Cc, w=Cc)
    elif out_layout == "hwdc":
        shape = (N, Ho, Wo, Do, Cc)
        os_ = dict(n=Do * Ho * Wo * Cc, c=1, d=Cc, h=Wo * Do * Cc, w=Do * Cc)
    else:
        raise ValueError(out_layout)
    out = torch.empty(shape, dtype=torch.float32, device=inp.device) if want_f32 else None
    sp = Split.empty(shape, inp.device, planes) if want_split else None
    if N == 0 or Do * Ho * Wo == 0:
        # empty batch / empty lattice: F.grid_sample returns an empty tensor; nothing to launch
        if want_f32 and want_split:
            return out, sp
        return out if want_f32 else sp
    d = L.GridSample3dDesc(_p(inp), 1 if in_layout == "cl" else 0, N, Cc, Di, Hi, Wi, _p(grid), _p(theta), Do, Ho, Wo,
                           _p(out), _p(sp.hi) if sp else None, _p(sp.lo) if sp else None, os_["n"], os_["c"],
                           os_["d"], os_["h"], os_["w"], _p(sp.lo2) if sp else None,
                           1 if (sp is not None and sp.f16) else 0, sp.scale if (sp is not None and sp.f16) else 0.0)
    L.call("emo_grid_sample3d", C.byref(d), _stream())
    if want_f32 and want_split:
        return out, sp
    return out if want_f32 else sp


def grid_sample2d_affine(img: torch.Tensor, theta: torch.Tensor, out_hw, mean=None, std=None, c_pad: int = 4,
                         want_nchw: bool = False):
    _chk(img); _chk(theta)
    N, Cc, Hi, Wi = img.shape
    Ho, Wo = out_hw
    out = torch.empty((N, 1, Ho, Wo, c_pad), dtype=torch.float32, device=img.device)
    nchw = torch.empty((N, Cc, Ho, Wo), dtype=torch.float32, device=img.device) if want_nchw else None
    d = L.GridSample2dAffineDesc(_p(img), N, Cc, Hi, Wi, _p(theta), Ho, Wo, _p(mean), _p(std), _p(out), c_pad, _p(nchw))
    L.call("emo_grid_sample2d_affine", C.byref(d), _stream())
    return (out, nchw) if want_nchw else out


def resize_bilinear(img: torch.Tensor, out_hw, mean=None, std=None, c_pad: int = 4):
    _chk(img)
    N, Cc, Hi, Wi = img.shape
    Ho, Wo = out_hw
    out = torch.empty((N, 1, Ho, Wo, c_pad), dtype=torch.float32, device=img.device)
    d = L.ResizeBilinearDesc(_p(img), N, Cc, Hi, Wi, Ho, Wo, _p(mean), _p(std), _p(out), c_pad)
    L.call("emo_resize_bilinear", C.byref(d), _stream())
    return out


# ------------------------------------------------------------------------------------------------
# GroupNorm pieces
# ------------------------------------------------------------------------------------------------
_ARENA = {}
_SLOT = 0  # which set of per-pass scratch (statistics arena, split-K workspace) the calls below use


def _dev_key(device):
    """Canonical (index-resolved) key of a CUDA device: torch.device('cuda') and tensor.device ('cuda:0') must name the
    same scratch — begin_pass() is called with the model's device, new_stats() with a tensor's."""
    d = torch.device(device)
    if d.type != "cuda":
        return (d.type, -1)
    return ("cuda", d.index if d.index is not None else torch.cuda.current_device())


def set_slot(k: int) -> int:
    """Select the scratch set for subsequent passes.  Passes that may be in flight at the same time on different streams
    (infer.DriverPipeline keeps several driver frames in flight) must not share the statistics arena or the
    self-cleaning split-K workspace, so each in-flight frame is issued under its own slot."""
    global _SLOT
    prev, _SLOT = _SLOT, int(k)
    return prev

_ARENA_SLOT = 2 * 32 * 2  # doubles per slot: up to N=2 samples x 32 groups x (sum, sumsq)


def begin_pass(device, slots: int = 384):
    """Start a source/driver pass: ONE memset zeroes the whole GroupNorm-statistics arena; new_stats() then hands out
    slices of it instead of launching a fill kernel per normalisation (57 per driver frame otherwise)."""
    key = (_dev_key(device), _SLOT)
    ar = _ARENA.get(key)
    if ar is None or ar["buf"].shape[0] < slots:
        ar = {"buf": torch.zeros((slots, _ARENA_SLOT), dtype=torch.float64, device=device), "idx": 0}
        _ARENA[key] = ar
    ar["buf"].zero_()
    ar["idx"] = 0


def new_stats(N: int, G: int, device) -> torch.Tensor:
    ar = _ARENA.get((_dev_key(device), _SLOT))
    if ar is not None and N * G * 2 <= _ARENA_SLOT and ar["idx"] < ar["buf"].shape[0]:
        t = ar["buf"][ar["idx"]][: N * G * 2].view(N, G, 2)
        ar["idx"] += 1
        return t
    return torch.zeros((N, G, 2), dtype=torch.float64, device=device)


def gn_stats(x: torch.Tensor, G: int = 32, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk(x)
    N, Cc = x.shape[0], x.shape[-1]
    S = x.numel() // (N * Cc)
    if stats is None:
        stats = new_stats(N, G, x.device)
    L.call("emo_gn_stats", _p(x), N, S, Cc, G, _p(stats), _stream())
    return stats


def gn_finalize(stats: torch.Tensor, count: float, gamma, beta, eps: float = 1e-5, ada_w=None, ada_b=None):
    N, G, _ = stats.shape
    Cc = gamma.numel()
    A = torch.empty((N, Cc), dtype=torch.float32, device=stats.device)
    B = torch.empty_like(A)
    d = L.GnFinalizeDesc(_p(stats), N, Cc, G, float(count), float(eps), _p(gamma), _p(beta), _p(ada_w), _p(ada_b),
                         _p(A), _p(B))
    L.call("emo_gn_finalize", C.byref(d), _stream())
    return A, B


def _apply_desc(x_ptr, shape, device, A=None, B=None, act: int = ACT_NONE, res=None, A2=None, B2=None, up: int = 1,
                want_f32: bool = False, want_split: bool = True, per_sample: bool = True, planes=2, gn=None):
    """emo_apply_desc + its freshly allocated outputs for a channels-last (N,D,H,W,C) input at `x_ptr`"""
    N, D, H, W, Cc = shape
    oshape = (N, D, H * up, W * up, Cc)
    out = torch.empty(oshape, dtype=torch.float32, device=device) if want_f32 else None
    sp = Split.empty(oshape, device, planes) if want_split else None
    d = L.ApplyDesc(x_ptr, N, Cc, D, H, W, _p(A), _p(B), 1 if per_sample else 0, _p(res), _p(A2), _p(B2), act, up,
                    _p(out), _p(sp.hi) if sp else None, _p(sp.lo) if sp else None, _p(sp.lo2) if sp else None,
                    _p(gn["stats"]) if gn else None, gn["stats"].shape[1] if gn else 0, float(gn["count"]) if gn else 0.0,
                    float(gn.get("eps", 1e-5)) if gn else 0.0, _p(gn["gamma"]) if gn else None, _p(gn["beta"]) if gn else None,
                    _p(gn.get("ada_w")) if gn else None, _p(gn.get("ada_b")) if gn else None,
                    1 if (sp is not None and sp.f16) else 0, sp.scale if (sp is not None and sp.f16) else 0.0)
    return d, out, sp


def apply(x: torch.Tensor, A=None, B=None, act: int = ACT_NONE, res=None, A2=None, B2=None, up: int = 1,
          want_f32: bool = False, want_split: bool = True, per_sample: bool = True, planes=2, gn=None):
    """y = act(x*A + B [+ res*A2 + B2]) on a channels-last (N,D,H,W,C) tensor; optional nearest x2 on (H, W).
    gn = dict(stats, count, gamma, beta[, ada_w, ada_b, eps]) fuses the GroupNorm finalisation (replaces A/B)."""
    _chk(x)
    d, out, sp = _apply_desc(_p(x), x.shape, x.device, A, B, act, res, A2, B2, up, want_f32, want_split, per_sample, planes, gn)
    L.call("emo_apply", C.byref(d), _stream())
    if want_f32 and want_split:
        return out, sp
    return out if want_f32 else sp


def gn_head(x: torch.Tensor, gn: dict, w: torch.Tensor, bias: Optional[torch.Tensor], act_out: int = ACT_NONE) -> torch.Tensor:
    """(N,D,H,W,C) fp32 channels-last -> (N,Cout,D,H,W): act_out(bias + w . relu(GroupNorm(x))) in one exact-fp32 pass
    (the image head, decoder.py:398-410).  w (Cout<=4, C) fp32, gn as in apply()."""
    _chk(x); _chk(w)
    N, D, H, W, Cc = x.shape
    Cout = w.shape[0]
    assert w.shape == (Cout, Cc) and 1 <= Cout <= 4
    out = torch.empty((N, Cout, D, H, W), dtype=torch.float32, device=x.device)
    d = L.GnHeadDesc(_p(x), N, Cc, D * H * W, _p(gn["stats"]), gn["stats"].shape[1], float(gn["count"]), float(gn.get("eps", 1e-5)),
                     _p(gn["gamma"]), _p(gn["beta"]), _p(w), _p(bias), Cout, act_out, _p(out))
    L.call("emo_gn_head", C.byref(d), _stream())
    return out


def split_bf16(x: torch.Tensor, planes=2) -> Split:
    """fp32 -> operand planes (bf16 x2 / x3, or fp16 x2 / x1 of x * F16_ACT_SCALE when planes == "h2" / "h1")"""
    _chk(x)
    sp = Split.empty(x.shape, x.device, planes)
    if sp.f16:
        L.call("emo_split_f16", _p(x), x.numel(), C.c_float(sp.scale), _p(sp.hi), _p(sp.lo), _stream())
    else:
        L.call("emo_split_bf16", _p(x), x.numel(), _p(sp.hi), _p(sp.lo), _p(sp.lo2), _stream())
    return sp


# ------------------------------------------------------------------------------------------------
# convolutions
# ------------------------------------------------------------------------------------------------
def _out_dim(i, k, s, p):
    return (i + 2 * p - k) // s + 1


_SPLITK_WS = {}


def _splitk_workspace(device) -> torch.Tensor:
    """Per-device (and per scratch slot, see set_slot) fp32 workspace for split-K convolutions.  It needs no initial state:
    each K part stores its partial sums to its own slice with plain stores, and the finalize / post kernels read only those
    slices and write nothing back.  Launches on one stream use it back to back, which is how the model issues its convs."""
    key = (_dev_key(device), _SLOT)
    if key not in _SPLITK_WS:
        _SPLITK_WS[key] = torch.zeros(2 * 1024 * 1024, dtype=torch.float32, device=device)
    return _SPLITK_WS[key]


class ConvProfiler:
    """CUDA-event bracket around every tensor-core conv launch (bench.py roofline evidence; off by default)."""

    def __init__(self):
        self.rec = []

    def summary(self):
        torch.cuda.synchronize()
        ms = sum(r[0].elapsed_time(r[1]) for r in self.rec)
        self.mma_flops = sum(r[2] * r[3] for r in self.rec)  # MMA flops actually issued (1, 3 or 6 per product)
        return ms, sum(r[2] for r in self.rec), len(self.rec)

    def table(self):
        """per-shape aggregate: (shape, launches, total ms, algorithmic TFLOP/s, MMA TFLOP/s)"""
        torch.cuda.synchronize()
        agg = {}
        for e0, e1, fl, passes, name in self.rec:
            a = agg.setdefault(name, [0, 0.0, 0.0, passes])
            a[0] += 1; a[1] += e0.elapsed_time(e1); a[2] += fl
        rows = [(k, v[0], v[1], v[2] / v[1] / 1e9, v[2] * v[3] / v[1] / 1e9) for k, v in agg.items()]
        return sorted(rows, key=lambda r: -r[2])


_conv_profiler: Optional[ConvProfiler] = None


def set_conv_profiler(p: Optional[ConvProfiler]):
    global _conv_profiler
    _conv_profiler = p


def _conv_desc(a: Split, w: PackedConvWeight, stride, pad, bias, residual, res_shift, act, post_add, out_nchw, stats, G, out,
               acc_chunk_mmas, split_k, upconv, post):
    """emo_conv_desc of one conv_igemm() call (with its freshly allocated output unless `out` is given), the value the call
    returns, the ctypes objects the descriptor points to, and the profiler label / algorithmic flops / MMA passes."""
    N, Di, Hi, Wi, Ci = a.shape
    assert Ci == w.cin, (Ci, w.cin)
    ws = None if not split_k else _splitk_workspace(a.hi.device)
    three = a.lo2 is not None
    assert not three or w.lo2 is not None, "3-plane activations need 3-plane weights (pack_conv_weight(planes=3))"
    assert a.f16 == w.f16, "fp16-plane activations need fp16-plane weights (pack_conv_weight(planes='h2')) and vice versa"
    one = a.lo is None
    assert one == (w.lo is None), "one-plane activations need one-plane weights (planes='h1') and vice versa"
    assert not (a.f16 and upconv and not one), "the sub-pixel convolution runs with two bf16 planes or one fp16 plane"
    kd, kh, kw = w.k
    if pad is None:
        pad = (kd // 2, kh // 2, kw // 2)
    Do, Ho, Wo = _out_dim(Di, kd, stride[0], pad[0]), _out_dim(Hi, kh, stride[1], pad[1]), _out_dim(Wi, kw, stride[2], pad[2])
    if upconv:
        assert w.hi.shape[0] == 16 and (kd, kh, kw) == (1, 3, 3) and tuple(stride) == (1, 1, 1) and Di == 1, "upconv needs pack_upconv_weight()"
        Ho, Wo = 2 * Hi, 2 * Wi
    if out is None:
        shape = (N, w.cout, Do, Ho, Wo) if out_nchw else (N, Do, Ho, Wo, w.cout)
        out = torch.empty(shape, dtype=torch.float32, device=a.hi.device)
    d = L.ConvDesc(_p(a.hi), _p(a.lo), N, Di, Hi, Wi, Ci, _p(w.hi), _p(w.lo), w.cout, w.cout_pad, kd, kh, kw,
                   stride[0], stride[1], stride[2], pad[0], pad[1], pad[2], Do, Ho, Wo, _p(bias), _p(residual),
                   res_shift, act, _p(post_add), _p(out), 1 if out_nchw else 0, _p(stats),
                   G if stats is not None else 0, _p(a.lo2) if three else None, _p(w.lo2) if three else None,
                   acc_chunk_mmas or w.acc_chunk, _p(ws), ws.numel() if ws is not None else 0, 1 if upconv else 0,
                   1 if a.f16 else 0, 1.0 / (a.scale * w.scale) if a.f16 else 0.0, None)
    ret, pd = out, None
    if post is not None:
        assert not out_nchw and not upconv, "post-op: channels-last output of a plain convolution"
        pkw = dict(post)
        if pkw.get("gn") is not None:
            assert stats is not None and pkw["gn"]["stats"] is stats, "a GroupNorm post-op uses the convolution's own statistics"
        pd, pout, psp = _apply_desc(None, (N, Do, Ho, Wo, w.cout), a.hi.device, **pkw)
        d.post = C.cast(C.pointer(pd), C.c_void_p)
        wf, wsp = pkw.get("want_f32", False), pkw.get("want_split", True)
        ret = (pout, psp) if (wf and wsp) else (pout if wf else psp)
    # algorithmic flops of the convolution being computed; MMA passes actually issued per algorithmic product
    # (sub-pixel mode issues 4 of the 9 taps)
    prof = (2.0 * N * Do * Ho * Wo * w.cout * Ci * kd * kh * kw, (6 if three else 1 if one else 3) * (4.0 / 9.0 if upconv else 1.0),
            f"{N}x{Di}x{Hi}x{Wi}x{Ci}->{w.cout} k{kd}{kh}{kw} s{stride[1]} p{('h1' if one else 'h2') if a.f16 else (3 if three else 2)}"
            + (" up2-subpixel" if upconv else ""))
    return d, ret, pd, prof


def conv_igemm(a: Split, w: PackedConvWeight, stride=(1, 1, 1), pad=None, bias=None, residual=None, res_shift: int = 0,
               act: int = ACT_NONE, post_add=None, out_nchw: bool = False, stats: Optional[torch.Tensor] = None,
               G: int = 32, out: Optional[torch.Tensor] = None, acc_chunk_mmas: int = 0, split_k: bool = True,
               upconv: bool = False, post: Optional[dict] = None):
    """upconv=True: `a` holds the LOW-resolution planes and `w` a pack_upconv_weight(): the result is
    conv3x3(pad 1)(nearest_x2(a)) at (2H, 2W), evaluated in sub-pixel form (see emo_conv_desc.upconv).
    post = dict(<arguments of apply()>): the elementwise pass that follows the convolution (GroupNorm / affine + residual +
    activation -> fp32 and/or operand planes; a `gn` post-op normalises with this convolution's `stats`).  Small split-K layers
    run it inside the finalize step (one launch instead of three, emo_conv_desc.post).  With `post` the call returns what
    apply() would return for it; the raw convolution output is then an internal scratch tensor."""
    d, ret, _pd, prof = _conv_desc(a, w, stride, pad, bias, residual, res_shift, act, post_add, out_nchw, stats, G, out,
                                   acc_chunk_mmas, split_k, upconv, post)
    if _conv_profiler is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        L.call("emo_conv_igemm", C.byref(d), _stream())
        e1.record()
        _conv_profiler.rec.append((e0, e1) + prof)
    else:
        L.call("emo_conv_igemm", C.byref(d), _stream())
    return ret


def conv_plan(a: Split, w: PackedConvWeight, stride=(1, 1, 1), pad=None, bias=None, residual=None, res_shift: int = 0,
              act: int = ACT_NONE, post_add=None, out_nchw: bool = False, stats: Optional[torch.Tensor] = None,
              G: int = 32, out: Optional[torch.Tensor] = None, acc_chunk_mmas: int = 0, split_k: bool = True,
              upconv: bool = False, post: Optional[dict] = None, sm_count: Optional[int] = None) -> L.ConvPlanInfo:
    """The launch plan conv_igemm() would run for the same arguments on a device of `sm_count` SMs (default: the current
    device's).  Nothing is launched; raises lib.EmoError where conv_igemm would refuse the arguments."""
    d, _ret, _pd, _prof = _conv_desc(a, w, stride, pad, bias, residual, res_shift, act, post_add, out_nchw, stats, G, out,
                                     acc_chunk_mmas, split_k, upconv, post)
    if sm_count is None:
        sm_count = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    lib = L.load()
    info = L.ConvPlanInfo()
    rc = lib.emo_conv_plan(C.byref(d), int(sm_count), C.byref(info))
    if rc != 0:
        raise L.EmoError(f"emo_conv_plan failed ({rc}): {lib.emo_last_error().decode()}")
    return info


def conv_direct(x: torch.Tensor, w: torch.Tensor, stride: int, pad: int, bias=None, stats=None, G: int = 32):
    """x (N,1,H,W,Cin_pad) fp32 channels-last; w (kh,kw,Cin_pad,Cout) fp32."""
    _chk(x); _chk(w)
    N, _, Hi, Wi, Cp = x.shape
    kh, kw, Cp2, Co = w.shape
    assert Cp == Cp2
    Ho, Wo = _out_dim(Hi, kh, stride, pad), _out_dim(Wi, kw, stride, pad)
    out = torch.empty((N, 1, Ho, Wo, Co), dtype=torch.float32, device=x.device)
    d = L.ConvDirectDesc(_p(x), N, Hi, Wi, Cp, _p(w), Co, kh, kw, stride, pad, Ho, Wo, _p(bias), _p(out), _p(stats),
                         G if stats is not None else 0)
    L.call("emo_conv_direct", C.byref(d), _stream())
    return out


STEM_CIN = 32   # channels of stem_pack()'s plane: 7 horizontal taps x 4 padded RGB channels, then 4 zero channels


def stem_pack(x4: torch.Tensor) -> Split:
    """x4 (N,1,H,W,4) fp32 channels-last (the padded RGB of resize_bilinear) -> one fp16 plane (N,1,H,W,32) of the 7x7 stem's
    horizontal taps: channel kx*4 + c = fp16(16 x[n, h, w + kx - 3, c]), zero outside the image and in channels 28..31.  The
    stem then runs on the tensor cores as conv_igemm(stem_pack(x4), pack_stem_weight(w), pad=(0, 3, 0)): a 7x1 convolution."""
    _chk(x4)
    N, D, H, W, Cc = x4.shape
    sp = Split.empty((N, D, H, W, STEM_CIN), x4.device, H1)
    L.call("emo_stem_pack", _p(x4), N * D, H, W, Cc, C.c_float(sp.scale), _p(sp.hi), _stream())
    return sp


def pack_stem_weight(w_direct: torch.Tensor, device=None) -> PackedConvWeight:
    """conv_direct weight of a 7x7 stem (7, 7, 4, Cout) [ky][kx][c][o] -> the one-plane weight of the 7x1 convolution over
    stem_pack()'s channels: [ky][Cout_pad][kx*4 + c] = fp16(256 w[ky][kx][c][o]), zero in channels 28..31."""
    kh, kw, cp, co = w_direct.shape
    assert (kh, kw, cp) == (7, 7, 4), w_direct.shape
    w = torch.zeros(co, STEM_CIN, kh, 1)
    w[:, :kw * cp, :, 0] = w_direct.detach().float().cpu().permute(3, 1, 2, 0).reshape(co, kw * cp, kh)
    return pack_conv_weight(w, device=device, planes=H1)


def linear(x: torch.Tensor, w: torch.Tensor, bias=None, add=None, scale: float = 1.0, act: int = ACT_NONE,
           x_strides=None, out: Optional[torch.Tensor] = None, out_strides=None, M=None, K=None):
    """out[m, n] = act((sum_k x[m,k] w[n,k] + bias[n] + add[m,n]) * scale); strides in elements."""
    _chk(w)
    Nn, Kk = w.shape
    if x_strides is None:
        assert x.dim() == 2 and x.is_contiguous()
        M, K = x.shape
        x_strides = (K, 1)
    assert K == Kk, (K, Kk)
    if out is None:
        out = torch.empty((M, Nn), dtype=torch.float32, device=w.device)
        out_strides = (Nn, 1)
    d = L.LinearDesc(_p(x), x_strides[0], x_strides[1], _p(w), _p(bias), _p(add), float(scale), act, M, Nn, Kk, _p(out),
                     out_strides[0], out_strides[1])
    L.call("emo_linear", C.byref(d), _stream())
    return out


# ------------------------------------------------------------------------------------------------
# resampling
# ------------------------------------------------------------------------------------------------
def upsample_trilinear(x: torch.Tensor, f=(2, 2, 2), add=None, stats=None, G: int = 32):
    _chk(x)
    N, D, H, W, Cc = x.shape
    out = torch.empty((N, D * f[0], H * f[1], W * f[2], Cc), dtype=torch.float32, device=x.device)
    d = L.ResampleDesc(_p(x), N, D, H, W, Cc, f[0], f[1], f[2], _p(add), _p(out), _p(stats), G if stats is not None else 0)
    L.call("emo_upsample_trilinear", C.byref(d), _stream())
    return out


def avgpool(x: torch.Tensor, f=(1, 2, 2), add=None, stats=None, G: int = 32):
    _chk(x)
    N, D, H, W, Cc = x.shape
    out = torch.empty((N, D // f[0], H // f[1], W // f[2], Cc), dtype=torch.float32, device=x.device)
    d = L.ResampleDesc(_p(x), N, D, H, W, Cc, f[0], f[1], f[2], _p(add), _p(out), _p(stats), G if stats is not None else 0)
    L.call("emo_avgpool", C.byref(d), _stream())
    return out


def maxpool2d_3x3s2(x: torch.Tensor):
    _chk(x)
    N, _, H, W, Cc = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.empty((N, 1, Ho, Wo, Cc), dtype=torch.float32, device=x.device)
    L.call("emo_maxpool2d_3x3s2", _p(x), N, H, W, Cc, _p(out), _stream())
    return out


def global_avgpool(x: torch.Tensor):
    _chk(x)
    N, Cc = x.shape[0], x.shape[-1]
    S = x.numel() // (N * Cc)
    out = torch.empty((N, Cc), dtype=torch.float32, device=x.device)
    L.call("emo_global_avgpool", _p(x), N, S, Cc, _p(out), _stream())
    return out


def pose_theta(srt: Optional[torch.Tensor], source_theta: Optional[torch.Tensor] = None, mix: bool = False,
               invert_warp: bool = False, mix_old: bool = False, theta_in: Optional[torch.Tensor] = None,
               smooth_state: Optional[torch.Tensor] = None, smooth_momentum: float = 0.5, smooth_init: bool = False,
               out: Optional[tuple] = None):
    """srt (N,9) [or theta_in (N,4,4)] -> theta (N,4,4), theta_warp (N,3,4), align2d (N,2,3). See emo_pose_theta.
    smooth_state (3,4) fp32 on device is updated in place (smooth_pose=True, notebooks/infer.py:571-581).
    out: (theta, theta_warp, align2d) buffers of those shapes to write instead of new tensors (a captured frame's pose)."""
    ref = srt if srt is not None else theta_in
    if ref is None:
        raise ValueError("pose_theta: srt or theta_in is required")
    for t in (srt, theta_in, source_theta, smooth_state):
        if t is not None:
            _chk(t)
    N = ref.shape[0]
    dev = ref.device
    if theta_in is not None and tuple(theta_in.shape) != (N, 4, 4):
        raise ValueError(f"pose_theta: theta_in must be (N,4,4), got {tuple(theta_in.shape)}")
    if smooth_state is not None and tuple(smooth_state.shape) != (3, 4):
        raise ValueError(f"pose_theta: smooth_state must be (3,4), got {tuple(smooth_state.shape)}")
    if out is None:
        theta = torch.empty((N, 4, 4), dtype=torch.float32, device=dev)
        warp = torch.empty((N, 3, 4), dtype=torch.float32, device=dev)
        align = torch.empty((N, 2, 3), dtype=torch.float32, device=dev)
    else:
        theta, warp, align = out
        for t, shp in zip(out, ((N, 4, 4), (N, 3, 4), (N, 2, 3))):
            _chk(t)
            if tuple(t.shape) != shp:
                raise ValueError(f"pose_theta: out must be (N,4,4), (N,3,4), (N,2,3), got {[tuple(o.shape) for o in out]}")
    d = pose_desc(N, _p(srt), _p(source_theta), _p(theta), _p(warp), _p(align), _p(theta_in), _p(smooth_state), mix=mix,
                  invert_warp=invert_warp, mix_old=mix_old, smooth_init=smooth_init, smooth_momentum=smooth_momentum)
    L.call("emo_pose_theta", C.byref(d), _stream())
    return theta, warp, align


def pose_desc(N: int, srt, source_theta, theta_out, theta_warp, align2d, theta_in=None, smooth_state=None, mix=False,
              invert_warp=False, mix_old=False, smooth_init=False, smooth_momentum: float = 0.5):
    """emo_pose_desc from raw pointers (int or None).  The state is smoothed as `theta * m + state * (1 - m)` on fp32
    tensors (notebooks/infer.py:577): torch rounds m to fp32, and 1 - m, evaluated by Python in double, to fp32 as well
    (as the c_float fields round them here)."""
    m = float(smooth_momentum)
    return L.PoseDesc(srt, source_theta, N, 1 if mix else 0, 1 if invert_warp else 0, theta_out, theta_warp, align2d, theta_in,
                      1 if mix_old else 0, 1 if smooth_init else 0, smooth_state, m, 1.0 - m)


def u8_to_image(u8_nhwc: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """uint8 (N,H,W,C) on device (PIL / numpy layout) -> fp32 (N,C,H,W) = u / 255 (ToTensor, notebooks/infer.py:229-243)"""
    _chk(u8_nhwc, torch.uint8)
    N, H, W, Cc = u8_nhwc.shape
    if out is None:
        out = torch.empty((N, Cc, H, W), dtype=torch.float32, device=u8_nhwc.device)
    L.call("emo_u8_to_image", _p(u8_nhwc), N, H, W, Cc, _p(out), _stream())
    return out


def image_to_u8(img_nchw: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 (N,C,H,W) -> uint8 (N,H,W,C) = trunc(clamp(x,0,1)*255): `.clamp(0,1)` + ToPILImage (notebooks/infer.py:641-644)"""
    _chk(img_nchw)
    N, Cc, H, W = img_nchw.shape
    if out is None:
        out = torch.empty((N, H, W, Cc), dtype=torch.uint8, device=img_nchw.device)
    L.call("emo_image_to_u8", _p(img_nchw), N, Cc, H, W, _p(out), _stream())
    return out


def s2_prepare(img_nchw: torch.Tensor, size: int, fast: bool):
    """The stage-2 input of a stage-1 image (N,3,h,w) fp32 in one pass: (resized (N,3,S,S) fp32 NCHW, the stem's operand).
    resized is resize_bilinear(img, (S, S)) as NCHW; the operand is that resize_bilinear output (N,1,S,S,4) itself, or with
    `fast` stem_pack() of it (one fp16 plane (N,1,S,S,32)).  Same bits as the two-step path."""
    _chk(img_nchw)
    N, Cc, Hi, Wi = img_nchw.shape
    assert Cc == 3, img_nchw.shape
    resized = torch.empty((N, 3, size, size), dtype=torch.float32, device=img_nchw.device)
    if fast:
        stem_in = Split.empty((N, 1, size, size, STEM_CIN), img_nchw.device, H1)
        x4, plane, scale = None, stem_in.hi, stem_in.scale
    else:
        stem_in = x4 = torch.empty((N, 1, size, size, 4), dtype=torch.float32, device=img_nchw.device)
        plane, scale = None, 0.0
    L.call("emo_s2_prepare", _p(img_nchw), N, Hi, Wi, size, _p(resized), _p(x4), _p(plane), C.c_float(scale), _stream())
    return resized, stem_in


def _stem_operand(N: int, size: int, fast: bool, device):
    """an empty stem operand of stage 2 at (N, size): (operand, x4, plane, scale) as the handoff entry points take them"""
    if fast:
        stem_in = Split.empty((N, 1, size, size, STEM_CIN), device, H1)
        return stem_in, None, stem_in.hi, stem_in.scale
    x4 = torch.empty((N, 1, size, size, 4), dtype=torch.float32, device=device)
    return x4, x4, None, 0.0


def s2_prepare_composite(img_nchw: torch.Tensor, matte: torch.Tensor, bg: torch.Tensor, size: int, fast: Optional[bool],
                         threshold: float = 0.3):
    """s2_prepare of composite(img, matte, bg, threshold) in one pass, the composited image never in memory: (resized, the stem's
    operand, or None with fast=None, when the stem reads s2_masked_stem's operand instead).  img (N,3,h,w), matte (N,1,h,w),
    bg (3,h,w) fp32.  Same bits as the two-step path."""
    _chk(img_nchw); _chk(matte); _chk(bg)
    N, Cc, Hi, Wi = img_nchw.shape
    assert Cc == 3 and tuple(matte.shape) == (N, 1, Hi, Wi) and tuple(bg.shape) == (3, Hi, Wi), (img_nchw.shape, matte.shape, bg.shape)
    resized = torch.empty((N, 3, size, size), dtype=torch.float32, device=img_nchw.device)
    stem_in, x4, plane, scale = (None, None, None, 0.0) if fast is None else _stem_operand(N, size, fast, img_nchw.device)
    L.call("emo_s2_prepare_composite", _p(img_nchw), _p(matte), _p(bg), C.c_float(threshold), N, Hi, Wi, size, _p(resized), _p(x4),
           _p(plane), C.c_float(scale), _stream())
    return resized, stem_in


def s2_masked_stem(resized: torch.Tensor, matte: torch.Tensor, fast: bool, out=None):
    """The stage-2 stem's operand of resized * matte (Stage2Model.forward's x4 * mask): resize_bilinear's (N,1,S,S,4) layout
    (R m, G m, B m, 0 m), or with `fast` stem_pack() of it.  resized (N,3,S,S), matte (N,1,S,S) fp32.  out: an operand of
    that kind to write in place.  Same bits as torch's product (then ops.stem_pack)."""
    _chk(resized); _chk(matte)
    N, Cc, S, S2 = resized.shape
    assert Cc == 3 and S == S2 and tuple(matte.shape) == (N, 1, S, S), (resized.shape, matte.shape)
    if out is None:
        stem_in, x4, plane, scale = _stem_operand(N, S, fast, resized.device)
    elif fast:
        stem_in, x4, plane, scale = out, None, out.hi, out.scale
    else:
        stem_in, x4, plane, scale = out, out, None, 0.0
    L.call("emo_s2_masked_stem", _p(resized), _p(matte), N, S, _p(x4), _p(plane), C.c_float(scale), _stream())
    return stem_in


def s2_finish_masked(resized: torch.Tensor, add: torch.Tensor, matte: torch.Tensor, face: Optional[torch.Tensor] = None,
                     out: Optional[torch.Tensor] = None, u8: Optional[torch.Tensor] = None):
    """(ffhq, u8): ffhq = (resized + add * (matte * face)).clamp_(0, 1) (N,3,H,W) fp32, Stage2Model.forward's masked residual,
    and u8 = image_to_u8(ffhq), in one pass.  matte (N,1,H,W) fp32; face (N,1,H,W) uint8 0 / 1 (parsing_masks' first mask) or
    None (cloth: matte alone)."""
    _chk(resized); _chk(add); _chk(matte)
    N, Cc, H, W = resized.shape
    assert Cc == 3 and add.shape == resized.shape and tuple(matte.shape) == (N, 1, H, W), (resized.shape, add.shape, matte.shape)
    if face is not None:
        _chk(face, torch.uint8)
        assert tuple(face.shape) == (N, 1, H, W), face.shape
    if out is None:
        out = torch.empty_like(resized)
    if u8 is None:
        u8 = torch.empty((N, H, W, 3), dtype=torch.uint8, device=resized.device)
    _chk(out); _chk(u8, torch.uint8)
    assert out.shape == resized.shape and tuple(u8.shape) == (N, H, W, 3), (out.shape, u8.shape)
    L.call("emo_s2_finish_masked", _p(resized), _p(add), _p(matte), _p(face), N, H, W, _p(out), _p(u8), _stream())
    return out, u8


def s2_finish(resized: torch.Tensor, add: torch.Tensor, out: Optional[torch.Tensor] = None,
              u8: Optional[torch.Tensor] = None):
    """(ffhq, u8): ffhq = (resized + add).clamp_(0, 1) (N,3,H,W) fp32 and u8 = image_to_u8(ffhq) (N,H,W,3), in one pass"""
    _chk(resized); _chk(add)
    N, Cc, H, W = resized.shape
    assert Cc == 3 and add.shape == resized.shape, (resized.shape, add.shape)
    if out is None:
        out = torch.empty_like(resized)
    if u8 is None:
        u8 = torch.empty((N, H, W, 3), dtype=torch.uint8, device=resized.device)
    _chk(out); _chk(u8, torch.uint8)
    assert out.shape == resized.shape and tuple(u8.shape) == (N, H, W, 3), (out.shape, u8.shape)
    L.call("emo_s2_finish", _p(resized), _p(add), N, H, W, _p(out), _p(u8), _stream())
    return out, u8


def resize_bicubic(img_nchw: torch.Tensor, out_hw) -> torch.Tensor:
    """F.interpolate(mode='bicubic', align_corners=False) (notebooks/infer.py:399-403, 551-556)"""
    _chk(img_nchw)
    N, Cc, Hi, Wi = img_nchw.shape
    out = torch.empty((N, Cc, out_hw[0], out_hw[1]), dtype=torch.float32, device=img_nchw.device)
    L.call("emo_resize_bicubic", _p(img_nchw), N, Cc, Hi, Wi, out_hw[0], out_hw[1], _p(out), _stream())
    return out


def composite(img: torch.Tensor, mask: torch.Tensor, bg: torch.Tensor, threshold: float = 0.3) -> torch.Tensor:
    """m' = where(mask > threshold, mask, 0) ** 8;  m' * img + (1 - m') * bg   (E_emo_infer_video.ipynb cell 41)
    img (N,C,H,W), mask (N,1,H,W), bg (C,H,W) fp32 on device."""
    _chk(img); _chk(mask); _chk(bg)
    N, Cc, H, W = img.shape
    assert mask.shape == (N, 1, H, W) and bg.shape == (Cc, H, W), (mask.shape, bg.shape)
    out = torch.empty_like(img)
    L.call("emo_composite", _p(img), _p(mask), _p(bg), N, Cc, H, W, C.c_float(threshold), _p(out), _stream())
    return out


def l2_flush(buf: torch.Tensor, clean: bool = False):
    """Benchmark helper: evict L2 by writing `buf` (>= 2x the L2 size).  clean=True also reads it back, so that L2 holds clean
    foreign lines and the kernel under test does not pay for the write-back of the flush's own dirty lines."""
    L.call("emo_l2_flush_clean" if clean else "emo_l2_flush", _p(buf), buf.numel() * buf.element_size(), _stream())


# ------------------------------------------------------------------------------------------------------------------
# mask pre/post-processing around the external mask networks (csrc/masks.cu)
# ------------------------------------------------------------------------------------------------------------------
def parsing_prepare(img_nchw: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, out_hw=(512, 512)) -> torch.Tensor:
    """(x - mean) / std per channel, then F.interpolate(size=out_hw, mode='bilinear')  (face_parcing.py:57-58)"""
    _chk(img_nchw); _chk(mean); _chk(std)
    N, Cc, Hi, Wi = img_nchw.shape
    out = torch.empty((N, Cc, out_hw[0], out_hw[1]), dtype=torch.float32, device=img_nchw.device)
    L.call("emo_parsing_prepare", _p(img_nchw), N, Cc, Hi, Wi, out_hw[0], out_hw[1], _p(mean), _p(std), _p(out), _stream())
    return out


def parsing_masks(logits_nchw: torch.Tensor, out_hw, label_sets, want_labels: bool = False):
    """F.interpolate(logits, size=out_hw, 'bilinear') -> argmax over classes -> membership in the four label sets
    (face_parcing.py:60-80) in one pass.  label_sets: four iterables of class ids.  Returns uint8 (4, N, 1, H, W) [, labels (N,1,H,W)]."""
    _chk(logits_nchw)
    N, K, Hi, Wi = logits_nchw.shape
    assert len(label_sets) == 4 and K <= 32
    bits = (C.c_uint * 4)(*[sum(1 << int(i) for i in set(ls)) for ls in label_sets])
    out = torch.empty((4, N, 1, out_hw[0], out_hw[1]), dtype=torch.uint8, device=logits_nchw.device)
    labels = torch.empty((N, 1, out_hw[0], out_hw[1]), dtype=torch.uint8, device=logits_nchw.device) if want_labels else None
    L.call("emo_parsing_masks", _p(logits_nchw), N, K, Hi, Wi, out_hw[0], out_hw[1], bits, _p(out), _p(labels), _stream())
    return (out, labels) if want_labels else out


def resize_area(img_nchw: torch.Tensor, out_hw, scale: float = 1.0, shift: float = 0.0) -> torch.Tensor:
    """F.interpolate(x * scale + shift, size=out_hw, mode='area') (adaptive average pooling; notebooks/infer.py:676, 682)"""
    _chk(img_nchw)
    N, Cc, Hi, Wi = img_nchw.shape
    out = torch.empty((N, Cc, out_hw[0], out_hw[1]), dtype=torch.float32, device=img_nchw.device)
    L.call("emo_resize_area", _p(img_nchw), N, Cc, Hi, Wi, out_hw[0], out_hw[1], float(scale), float(shift), _p(out), _stream())
    return out


# ------------------------------------------------------------------------------------------------------------------
# image plumbing of the demo video loop (csrc/video.cu)
# ------------------------------------------------------------------------------------------------------------------
def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def _bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


# Pillow's LANCZOS and BICUBIC filters (libImaging/Resample.c) with their supports: the only two the video loop uses
RESAMPLE_FILTERS = {"lanczos": (_lanczos, 3.0), "bicubic": (_bicubic, 2.0)}
RESAMPLE_BITS = 22   # Pillow's PRECISION_BITS: fixed-point coefficients of uint8 resizes


def resample_coeffs(in_size: int, out_size: int, filter: str):
    """Pillow's fixed-point taps of a resize of one axis from in_size to out_size (precompute_coeffs over the box (0, in_size),
    then normalize_coeffs_8bpc): a list of (first tap, [coefficients]) per output index.  Python floats and math.sin are the
    IEEE double operations and the libm of Pillow's C code, so these are Pillow's integers."""
    fn, support = RESAMPLE_FILTERS[filter]
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = support * fs
    ss = 1.0 / fs
    one = 1 << RESAMPLE_BITS
    taps = []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        k = [fn((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        taps.append((xmin, [int(-0.5 + w * one) if w < 0 else int(0.5 + w * one) for w in k]))
    return taps


@dataclass
class ResampleTaps:
    """resample_coeffs() of one axis on the device as emo_resample_u8 reads it: int32 (out, 2 + kmax) rows of (first tap, tap
    count, coefficients); lo / hi: the first and one past the last input index any output reads (Pillow's ybox)."""
    table: torch.Tensor
    kmax: int
    lo: int
    hi: int


_RESAMPLE_TAPS = {}


def resample_taps(in_size: int, out_size: int, filter: str, device) -> ResampleTaps:
    """The cached device taps of (in_size -> out_size, filter).  The first call builds and uploads them, so a caller that
    captures resample_u8 calls this for its shapes first: a captured launch must not copy from the host."""
    if filter not in RESAMPLE_FILTERS:
        raise ValueError(f"filter={filter!r}: one of {sorted(RESAMPLE_FILTERS)}")
    key = (int(in_size), int(out_size), filter, _dev_key(device))
    t = _RESAMPLE_TAPS.get(key)
    if t is None:
        coeffs = resample_coeffs(int(in_size), int(out_size), filter)
        kmax = max(len(k) for _, k in coeffs)
        rows = [[first, len(k)] + k + [0] * (kmax - len(k)) for first, k in coeffs]
        table = torch.tensor(rows, dtype=torch.int32)
        t = ResampleTaps(table if L.DRY_RUN else table.to(device), kmax, coeffs[0][0], coeffs[-1][0] + len(coeffs[-1][1]))
        _RESAMPLE_TAPS[key] = t
    return t


def _u8_image(t: torch.Tensor, what: str):
    """(H, W, 3) uint8 on the device with rows of any pitch and packed pixels -> its row pitch in bytes"""
    assert (t.is_cuda or L.DRY_RUN) and t.dtype == torch.uint8 and t.dim() == 3 and t.shape[2] == 3, (what, t.shape, t.dtype)
    assert t.stride(2) == 1 and t.stride(1) == 3 and t.stride(0) >= 3 * t.shape[1], (what, t.stride())
    return t.stride(0)


def resample_u8(src: torch.Tensor, size, filter: str, crop=None, dst: Optional[torch.Tensor] = None, src_bgr: bool = False,
                dst_bgr: bool = False) -> torch.Tensor:
    """Pillow's Image.crop(crop).resize(size, filter) of a (H, W, 3) uint8 image on the device, bit for bit: filter "lanczos"
    (Image.LANCZOS) or "bicubic" (Image.BICUBIC), size = (width, height) as Pillow takes it, crop = integer (left, upper,
    right, lower) or None for the whole image; pixels outside the source read as 0.  src and dst may be views with any row
    pitch (a panel of a wider row); src_bgr / dst_bgr give each side's channel order.  Returns dst, (height, width, 3)."""
    sp = _u8_image(src, "src")
    H, W = src.shape[:2]
    x0, y0, x1, y1 = (0, 0, W, H) if crop is None else tuple(crop)
    if not all(isinstance(v, numbers.Integral) for v in (x0, y0, x1, y1)) or x1 <= x0 or y1 <= y0:
        raise ValueError(f"crop must be a non-empty box of integers (left, upper, right, lower), got {crop}")
    ow, oh = int(size[0]), int(size[1])
    if ow <= 0 or oh <= 0:
        raise ValueError(f"size must be positive (width, height), got {size}")
    cw, ch = x1 - x0, y1 - y0
    if dst is None:
        dst = torch.empty((oh, ow, 3), dtype=torch.uint8, device=src.device)
    dp = _u8_image(dst, "dst")
    assert tuple(dst.shape[:2]) == (oh, ow), (dst.shape, size)
    ht = resample_taps(cw, ow, filter, src.device) if ow != cw else None
    vt = resample_taps(ch, oh, filter, src.device) if oh != ch else None
    tmp, t0, rows = None, 0, 0
    if ht is not None and vt is not None:
        t0, rows = vt.lo, vt.hi - vt.lo
        tmp = torch.empty((rows, ow, 3), dtype=torch.uint8, device=src.device)
    x0, y0 = int(x0), int(y0)
    L.call("emo_resample_u8", _p(src), H, W, sp, int(src_bgr), x0, y0, cw, ch, _p(dst), oh, ow, dp, int(dst_bgr),
           _p(ht.table) if ht else None, ht.kmax if ht else 0, _p(vt.table) if vt else None, vt.kmax if vt else 0, _p(tmp), t0, rows,
           _stream())
    return dst


def mask_dilate(m: torch.Tensor, thr: float, radius: int) -> torch.Tensor:
    """max over a (2 radius + 1)^2 window, clipped to the image, of (m >= thr): m (N,1,H,W) fp32 -> (N,1,H,W) fp32 0 / 1.  With
    radius 20 this is the notebook's cv2.dilate((m >= thr).float(), ones(21, 21), iterations=2) (cell 40)."""
    _chk(m)
    N, Cc, H, W = m.shape
    assert Cc == 1, m.shape
    out = torch.empty_like(m)
    tmp = torch.empty((N, H, W), dtype=torch.uint8, device=m.device)
    L.call("emo_mask_dilate", _p(m), N, H, W, C.c_float(thr), int(radius), _p(tmp), _p(out), _stream())
    return out
