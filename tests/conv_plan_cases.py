"""The case table of the implicit-GEMM convolution sweep, shared by tests/test_conv_plan_cpu.py (every case reaches the launch
plan it names, and the table as a whole reaches every configuration of the planner) and tests/test_conv_plan_gpu.py (every
case against float64).

A case is a convolution (shape + options of ops.conv_igemm) and the plan class it is meant to reach at 132 SMs (H100 SXM):
"<kernel instantiation> BN<N tile> <main loop> <finish>[ 3-D]", main loop "rr2" / "rr3" (row reuse with an A ring of 2 / 3
halo tiles) or "tap" (one {A, B} stage per tap), finish as emo_conv_plan_info.finish (lib.CONV_FINISH), " 3-D" for inputs of
depth > 1 (plan_class): a 2-D case does not sweep the depth halo, padding and tiles of a 3-D launch."""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
import torch
import torch.nn.functional as F

SM_COUNT = 132  # H100 SXM


@dataclass(frozen=True)
class Case:
    want: str                  # plan class at SM_COUNT SMs
    Cin: int
    Cout: int
    sp: tuple                  # input (H, W) or (D, H, W); the LOW-resolution map with upconv
    k: int = 3                 # kd = kh = kw (kd = 1 for 2-D maps), padding k // 2
    stride: int = 1
    planes: object = 2         # 2, 3 or "h2" (ops.H2)
    N: int = 1
    upconv: bool = False
    split_k: bool = True
    bias: bool = True
    residual: bool = False
    res_shift: int = 0
    act: int = 0               # lib.ACT_*
    post_add: bool = False
    out_nchw: bool = False
    stats: bool = False
    G: int = 32
    post: bool = False         # GroupNorm + ReLU post-op (emo_conv_desc.post) on the convolution's own statistics
    acc: int = 0               # acc_chunk_mmas (0: the packed weight's default)

    @property
    def id(self) -> str:
        opts = [k for k in ("upconv", "residual", "post_add", "out_nchw", "stats", "post") if getattr(self, k)]
        opts += [f"rs{self.res_shift}"] if self.res_shift else []
        opts += [f"act{self.act}"] if self.act else []
        opts += [f"acc{self.acc}"] if self.acc else []
        opts += ["nosplit"] if not self.split_k else []
        opts += [f"G{self.G}"] if self.stats and self.G != 32 else []
        sp = "x".join(map(str, self.sp))
        return f"N{self.N}-{self.Cin}-{self.Cout}-{sp}-k{self.k}s{self.stride}-p{self.planes}" + "".join("-" + o for o in opts)


B2, B3, H2 = 2, 3, "h2"
RELU, SIGMOID, TANH = 1, 2, 3

CASES = [
    # ---- the classes the shipped models reach (tests/test_conv_plan_cpu.py checks that this list covers them) ----
    # bf16 two planes, KC = 64
    Case("conv<64,2> BN128 rr2 none", 64, 128, (96, 96), residual=True, stats=True),
    Case("conv<64,2> BN128 rr2 apply", 64, 256, (64, 80), post=True, stats=True),
    Case("conv<64,2> BN128 tap none", 64, 128, (96, 96), k=1, post_add=True),
    Case("conv<64,2> BN128 tap finalize", 256, 256, (8, 8), residual=True, stats=True),
    Case("conv<64,2> BN128 tap finalize+apply", 128, 256, (24, 24), post=True, stats=True),
    Case("conv<64,2> BN96 rr3 none", 64, 96, (96, 96), act=TANH, stats=True),
    Case("conv<64,2> BN96 rr3 apply", 64, 96, (96, 96), post=True, stats=True),
    Case("conv<64,2> BN96 tap none", 64, 192, (96, 40), k=1, residual=True),
    Case("conv<64,2> BN80 rr3 none", 64, 160, (96, 40), residual=True, stats=True),
    Case("conv<64,2> BN80 rr3 apply", 64, 160, (96, 40), post=True, stats=True),
    Case("conv<64,2> BN80 tap none", 64, 160, (96, 40), k=1, out_nchw=True),
    Case("conv<64,2> BN64 rr3 none", 64, 64, (96, 96), stats=True),
    Case("conv<64,2> BN64 rr3 apply", 64, 64, (96, 96), post=True, stats=True),
    Case("conv<64,2> BN16 rr3 none", 64, 320, (16, 32), split_k=False, stats=True),            # BN 16 % cpg 10: per-column stats
    Case("conv<64,2> BN64 tap none", 64, 64, (96, 96), k=1, residual=True),
    Case("conv<64,2> BN32 rr3 none", 64, 32, (96, 96), stats=True, G=8),
    Case("conv<64,2> BN32 rr3 apply", 64, 32, (96, 96), post=True, stats=True),
    Case("conv<64,2> BN32 tap none", 64, 32, (96, 96), k=1, stats=True),
    # bf16 two planes, KC = 32 (Cin % 64 != 0)
    Case("conv<32,2> BN96 rr3 none", 96, 96, (96, 96), residual=True, res_shift=1, stats=True),
    Case("conv<32,2> BN96 rr3 apply", 160, 96, (96, 96), post=True, stats=True),
    Case("conv<32,2> BN96 tap none", 160, 96, (96, 96), k=1),
    Case("conv<32,2> BN80 rr3 none", 32, 160, (96, 40), residual=True, stats=True),
    Case("conv<32,2> BN80 rr3 apply", 32, 160, (96, 40), post=True, stats=True),
    Case("conv<32,2> BN32 rr3 none", 32, 32, (96, 96), residual=True, stats=True),
    Case("conv<32,2> BN16 tap none", 32, 3, (32, 32), k=1, act=SIGMOID, out_nchw=True, N=2),
    # sub-pixel up-convolution
    Case("ps<64,2> BN128 rr2 none", 64, 128, (48, 48), upconv=True, stats=True),
    Case("ps<64,2> BN96 rr3 none", 64, 96, (48, 48), upconv=True, residual=True, res_shift=1),
    Case("ps<64,2> BN80 rr3 none", 64, 160, (24, 40), upconv=True, residual=True, stats=True),
    Case("ps<64,2> BN64 rr3 none", 64, 64, (48, 40), upconv=True, post_add=True, stats=True),
    # fp16 two planes, KC = 64
    Case("f16<64,2> BN128 rr2 none", 64, 128, (96, 96), planes=H2, residual=True, stats=True),
    Case("f16<64,2> BN128 rr2 apply 3-D", 64, 256, (4, 16, 80), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN128 rr2 apply", 128, 256, (64, 80), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN128 tap none", 64, 128, (96, 96), k=1, planes=H2, post_add=True, stats=True),
    Case("f16<64,2> BN128 tap finalize", 512, 128, (4, 4), k=1, planes=H2, out_nchw=True),
    Case("f16<64,2> BN128 tap finalize+apply", 128, 128, (32, 32), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN128 tap post", 256, 256, (8, 8), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN96 rr3 none", 192, 96, (96, 96), planes=H2, residual=True),
    Case("f16<64,2> BN96 rr3 apply", 64, 192, (96, 40), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN96 tap none", 64, 192, (96, 40), k=1, planes=H2, stats=True),
    Case("f16<64,2> BN64 rr3 none", 64, 64, (96, 96), planes=H2, residual=True, stats=True),
    Case("f16<64,2> BN64 rr3 apply", 64, 64, (96, 96), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN64 tap none 3-D", 128, 64, (4, 64, 64), k=1, planes=H2),
    Case("f16<64,2> BN64 tap finalize+apply", 64, 64, (64, 64), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN64 tap post", 64, 64, (32, 32), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN32 rr3 apply 3-D", 64, 32, (8, 64, 64), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN32 tap none 3-D", 64, 32, (8, 64, 64), k=1, planes=H2, residual=True),
    Case("f16<64,2> BN32 tap none", 64, 256, (64, 64), k=1, planes=H2, split_k=False, stats=True),
    Case("f16<64,2> BN32 tap apply", 64, 32, (96, 96), k=1, planes=H2, post=True, stats=True),
    Case("f16<64,2> BN16 tap none", 256, 512, (8, 8), k=1, stride=2, planes=H2, residual=True),
    Case("f16<64,2> BN16 tap apply", 64, 64, (32, 32), k=1, planes=H2, post=True, stats=True),
    # fp16 two planes, KC = 32
    Case("f16<32,2> BN96 rr3 none 3-D", 96, 96, (4, 64, 64), planes=H2, residual=True, stats=True),
    Case("f16<32,2> BN96 rr3 apply 3-D", 96, 96, (4, 64, 64), planes=H2, post=True, stats=True),
    Case("f16<32,2> BN96 tap none 3-D", 96, 96, (4, 64, 64), k=1, planes=H2, out_nchw=True),
    Case("f16<32,2> BN32 rr3 none 3-D", 32, 32, (8, 64, 64), planes=H2, residual=True),
    Case("f16<32,2> BN16 rr3 none", 32, 3, (4, 16), planes=H2, split_k=False, post_add=True),
    # the 3-D layers of stage 1 in exact mode (Cin / Cout as the model's): volume blocks, U-Net, warp generator.  A 3-D per-tap
    # case tiles depth (td = 2 on 8 x 8 slices) with a depth the tile does not divide; row reuse keeps a tile in one depth
    # slice (td = 1), so its cases take an odd depth, whose first and last output slices read the depth padding.
    Case("f16<64,2> BN128 rr2 none 3-D", 384, 384, (5, 32, 32), planes=H2, residual=True, stats=True),
    Case("f16<64,2> BN128 tap none 3-D", 192, 384, (45, 8, 8), k=1, planes=H2, split_k=False),
    Case("f16<64,2> BN128 tap finalize 3-D", 256, 256, (7, 8, 8), planes=H2, residual=True, stats=True),
    Case("f16<64,2> BN128 tap finalize+apply 3-D", 512, 256, (5, 8, 8), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN96 rr3 none 3-D", 192, 192, (5, 32, 32), planes=H2, residual=True, stats=True),
    Case("f16<64,2> BN96 rr3 apply 3-D", 384, 192, (5, 32, 32), planes=H2, post=True, stats=True),
    Case("f16<64,2> BN96 tap none 3-D", 384, 192, (65, 8, 8), k=1, planes=H2, split_k=False),
    Case("f16<64,2> BN64 rr3 none 3-D", 64, 64, (9, 32, 32), planes=H2, residual=True, stats=True),
    Case("f16<64,2> BN64 rr3 apply 3-D", 128, 64, (9, 32, 32), planes=H2, post=True, stats=True),
    # the warp generator's head: tanh, then the identity grid added
    Case("f16<32,2> BN16 rr3 none 3-D", 32, 3, (5, 16, 24), planes=H2, split_k=False, act=TANH, post_add=True),

    # ---- configurations the models do not reach today ----
    # the other wgmma N widths (bf16 and fp16 have one instruction form per width)
    Case("conv<64,2> BN112 rr2 none", 64, 112, (96, 96), residual=True, stats=True, G=16),
    Case("conv<64,2> BN48 rr3 none", 64, 144, (64, 64), residual=True, stats=True, G=16),
    Case("f16<64,2> BN112 rr2 none", 64, 112, (96, 96), planes=H2, residual=True, stats=True, G=16),
    Case("f16<64,2> BN48 rr3 none", 64, 144, (64, 64), planes=H2, residual=True, stats=True, G=16),
    Case("f16<64,2> BN80 rr3 none", 64, 160, (96, 40), planes=H2, act=TANH, stats=True),
    Case("conv<64,2> BN16 tap none", 64, 16, (8, 16), k=1, split_k=False, stats=True, G=16),
    # three planes (fp32-faithful bf16)
    Case("conv<64,3> BN64 rr2 none", 64, 64, (96, 96), planes=B3, residual=True, stats=True),
    Case("conv<32,3> BN128 tap finalize 3-D", 512, 256, (8, 8, 8), planes=B3, residual=True, stats=True),
    Case("conv<64,3> BN16 tap none 3-D", 64, 64, (16, 16, 16), k=3, stride=2, planes=B3, split_k=False, residual=True, stats=True),
    Case("conv<32,3> BN96 rr3 none 3-D", 64, 96, (4, 48, 48), planes=B3, residual=True, stats=True),
    Case("conv<32,3> BN16 tap none 3-D", 96, 96, (8, 8, 8), planes=B3, split_k=False, residual=True, stats=True),
    # row reuse with KC = 32 although Cin % 64 == 0 (a 64-channel halo tile does not fit next to the B ring)
    Case("conv<32,2> BN128 rr3 none", 64, 1024, (2, 256), N=4, residual=True),
    Case("f16<32,2> BN128 rr3 none", 64, 1024, (2, 256), N=4, planes=H2, residual=True),
    Case("conv<32,3> BN16 rr2 none", 64, 128, (1, 128), planes=B3, split_k=False, stats=True),
    # split-K: post-add, NCHW output, odd Cout, batch of 2 with statistics
    Case("conv<64,2> BN128 tap finalize", 256, 128, (8, 8), post_add=True, act=TANH, stats=True, N=2),
    Case("conv<64,2> BN16 tap finalize", 512, 3, (16, 16), k=1, out_nchw=True, act=SIGMOID, N=2),
    Case("f16<64,2> BN64 tap post", 256, 64, (8, 8), planes=H2, post=True, stats=True, N=2),
    # items > grid in the per-tap loop, ragged boxes, odd Cout on the scalar path, explicit accumulation chunks
    Case("conv<64,2> BN16 tap none", 64, 5, (96, 200), k=1, residual=False, stats=True, G=5, acc=6),
    Case("conv<64,3> BN16 tap none", 64, 7, (40, 72), k=3, stride=2, planes=B3, split_k=False, out_nchw=True, acc=30, N=2),
    Case("f16<64,2> BN16 tap none 3-D", 64, 12, (20, 20, 20), k=3, stride=2, planes=H2, split_k=False, residual=True, stats=True, G=4, acc=9),
    Case("conv<32,3> BN128 tap none 3-D", 96, 256, (24, 24, 24), k=1, planes=B3, post_add=True),
    Case("f16<32,2> BN16 tap none", 32, 13, (72, 72), k=1, planes=H2, residual=True, acc=3),
    Case("conv<64,2> BN128 rr2 none", 64, 384, (80, 80), residual=True, res_shift=1, post_add=True, acc=40),
    Case("ps<64,2> BN128 rr2 none", 128, 256, (40, 56), upconv=True, residual=True, res_shift=1, stats=True, acc=36),
]


def plan_class(info, depth: int) -> str:
    """plan class of a convolution whose input has `depth` slices: " 3-D" follows the class of a volume (depth > 1), whose
    tiles meet the depth halo, depth padding and depth tiles that a 2-D map never reaches"""
    from emoportraits_b200 import lib as L

    loop = f"rr{info.sa}" if info.yreuse else "tap"
    return f"{L.conv_kernel_name(info.kernel)} BN{info.BN} {loop} {L.CONV_FINISH[info.finish]}" + (" 3-D" if depth > 1 else "")


def depth(c: Case) -> int:
    """input depth of a case (1 for a 2-D map)"""
    return c.sp[0] if len(c.sp) == 3 else 1


# ------------------------------------------------------------------------------------------------------------------
# operands and the float64 reference
# ------------------------------------------------------------------------------------------------------------------
def out_shape(c: Case):
    """(Do, Ho, Wo) of the convolution"""
    sp = c.sp if len(c.sp) == 3 else (1,) + tuple(c.sp)
    if c.upconv:
        return 1, 2 * sp[1], 2 * sp[2]
    kd = c.k if len(c.sp) == 3 else 1
    return tuple((i + 2 * (k // 2) - k) // c.stride + 1 for i, k in zip(sp, (kd, c.k, c.k)))


def make(c: Case, device, positive: bool = False):
    """Seeded float32 tensors of a case (NCDHW / NCHW, on `device`): x, w, bias, residual, post_add"""
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    nd = len(c.sp)
    x = torch.randn((c.N, c.Cin) + tuple(c.sp), generator=g)
    kshape = (c.k,) * nd
    w = torch.randn((c.Cout, c.Cin) + kshape, generator=g) / math.sqrt(c.Cin * c.k ** nd)
    if positive:
        x, w = x.abs(), w.abs()
    Do, Ho, Wo = out_shape(c)
    osp = (Do, Ho, Wo) if nd == 3 else (Ho, Wo)
    b = torch.randn(c.Cout, generator=g) if c.bias else None
    res = None
    if c.residual:
        rsp = osp[:-2] + (osp[-2] >> c.res_shift, osp[-1] >> c.res_shift)
        res = torch.randn((c.N, c.Cout) + rsp, generator=g)
    pa = torch.randn((1, c.Cout) + osp, generator=g) if c.post_add else None
    return [t.to(device) if t is not None else None for t in (x, w, b, res, pa)]


def cl(x):
    """NCHW / NCDHW -> channels-last (N, D, H, W, C)"""
    if x.dim() == 4:
        x = x[:, :, None]
    return x.permute(0, 2, 3, 4, 1).contiguous()


def reference(c: Case, x, w, b, res, pa):
    """float64 result of the case (NCDHW / NCHW) before the post-op, and the largest magnitude the kernel accumulates or adds
    on the way (the scale its rounding errors are relative to: an activation can shrink the output but not those errors)"""
    nd = len(c.sp)
    xd, wd = x.double(), w.double()
    if c.upconv:
        y = F.conv2d(F.interpolate(xd, scale_factor=2, mode="nearest"), wd, padding=1)
    else:
        y = (F.conv3d if nd == 3 else F.conv2d)(xd, wd, stride=c.stride, padding=c.k // 2)
    if b is not None:
        y = y + b.double().view((1, -1) + (1,) * nd)
    if res is not None:
        r = res.double()
        if c.res_shift:
            r = F.interpolate(r, scale_factor=(1, 2, 2) if nd == 3 else 2, mode="nearest")
        y = y + r
    scale = y.abs().max().item()
    if c.act == RELU:
        y = torch.relu(y)
    elif c.act == SIGMOID:
        y = torch.sigmoid(y)
    elif c.act == TANH:
        y = torch.tanh(y)
    if pa is not None:
        y = y + pa.double()
    return y, max(scale, y.abs().max().item())


def conv_args(c: Case, ops, x, w, b, res, pa, stats=None, out=None, acc=None):
    """(Split, PackedConvWeight, keyword arguments) of ops.conv_igemm / ops.conv_plan for the case"""
    planes = ops.H2 if c.planes == H2 else c.planes
    if c.upconv:
        pw = ops.pack_upconv_weight(w.cpu(), device=x.device)
    else:
        pw = ops.pack_conv_weight(w.cpu(), device=x.device, planes=planes)
    xs = cl(x)
    if x.is_cuda:
        a = ops.split_bf16(xs, planes)
    else:   # planning only: the operand values do not matter
        a = ops.Split.empty(xs.shape, x.device, planes)
    s3 = (c.stride,) * 3 if len(c.sp) == 3 else (1, c.stride, c.stride)
    kw = dict(stride=s3, bias=b, residual=cl(res) if res is not None else None, res_shift=c.res_shift, act=c.act,
              post_add=cl(pa)[0] if pa is not None else None, out_nchw=c.out_nchw, stats=stats, G=c.G, out=out,
              acc_chunk_mmas=c.acc if acc is None else acc, split_k=c.split_k, upconv=c.upconv)
    if c.post:
        Do, Ho, Wo = out_shape(c)
        gamma = torch.linspace(0.5, 1.5, c.Cout, device=x.device)
        beta = torch.linspace(-0.5, 0.5, c.Cout, device=x.device)
        kw["post"] = dict(act=ops.ACT_RELU, planes=planes, want_f32=True, want_split=False,
                          gn=dict(stats=stats, count=Do * Ho * Wo * c.Cout / c.G, gamma=gamma, beta=beta))
    return a, pw, kw


def post_reference(c: Case, y, G):
    """GroupNorm (gamma, beta as conv_args builds them) + ReLU of the float64 convolution output"""
    gamma = torch.linspace(0.5, 1.5, c.Cout, device=y.device, dtype=torch.float64)
    beta = torch.linspace(-0.5, 0.5, c.Cout, device=y.device, dtype=torch.float64)
    return torch.relu(F.group_norm(y, G, gamma, beta, 1e-5))
