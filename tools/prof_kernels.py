"""Representative launches of every roofline kernel for `ncu --set full` captures, e.g.
   ncu --set full -k regex:conv_igemm -o conv python tools/prof_kernels.py
   conv_igemm_kernel   decoder 3x3 512->512 @64^2 with residual (dominant layer), 3x3 128->128 @512^2 with
                       residual (row-reuse main loop), sub-pixel up-conv 192->128 @256^2 -> 512^2 (PS = true);
                       F16 = true: warp-generator 3x3x3 64->32 @32x64x64 (fp16 two-plane operands), ResNet-18 3x3 64->64
                       @32^2 (split-K)
   splitk_post_kernel  the fused finalize + GroupNorm + ReLU + plane split behind that split-K layer
   apply_kernel        GroupNorm-apply + ReLU + plane split @512^2 x 128
   gn_head_kernel      image head @512^2 x 128 -> 3
   gs3_cl_kernel       96ch 64^3 volume through a warp-field tensor / through the fused affine lattice; 16x64x64 (model-true)"""
import math, sys, pathlib
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import torch
from emoportraits_b200 import ops

dev = "cuda"
g = torch.Generator().manual_seed(0)


def conv(Cin, Cout, sp, k, planes, residual=True, upconv=False, post=False):
    three = len(sp) == 3
    shape = (1,) + (tuple(sp) if three else (1,) + tuple(sp)) + (Cin,)
    x = torch.randn(shape, generator=g).to(dev)
    w = torch.randn((Cout, Cin) + (k,) * len(sp), generator=g) / math.sqrt(Cin * k ** len(sp))
    pw = ops.pack_upconv_weight(w) if upconv else ops.pack_conv_weight(w, planes=planes)
    a = ops.split_bf16(x, planes)
    osp = tuple(2 * v for v in sp) if upconv else tuple(sp)
    oshape = (1,) + (osp if three else (1,) + osp) + (Cout,)
    res = torch.randn(oshape, generator=g).to(dev) if residual else None
    ops.begin_pass(dev)
    st = ops.new_stats(1, 32, dev)
    bias = torch.zeros(Cout, device=dev)
    kw = {}
    if post:
        kw["post"] = dict(gn=dict(stats=st, count=math.prod(osp) * Cout / 32, gamma=torch.ones(Cout, device=dev), beta=torch.zeros(Cout, device=dev)),
                          act=ops.ACT_RELU, planes=planes)
    for _ in range(3):
        ops.conv_igemm(a, pw, bias=bias, residual=res, stats=st, upconv=upconv, **kw)
    torch.cuda.synchronize()


conv(512, 512, (64, 64), 3, 2)
conv(128, 128, (512, 512), 3, 2)
conv(192, 128, (256, 256), 3, 2, residual=False, upconv=True)
conv(64, 32, (32, 64, 64), 3, "h2", residual=False)
conv(64, 64, (32, 32), 3, "h2", residual=False, post=True)

x = torch.randn(1, 1, 512, 512, 128, generator=g).to(dev)
ops.begin_pass(dev)
st = ops.gn_stats(x, 32)
gn = dict(stats=st, count=x.numel() / 32, gamma=torch.ones(128, device=dev), beta=torch.zeros(128, device=dev))
for _ in range(3):
    ops.apply(x, gn=gn, act=ops.ACT_RELU)
w, b = torch.randn(3, 128, device=dev), torch.zeros(3, device=dev)
for _ in range(3):
    ops.gn_head(x, gn, w, b, act_out=ops.ACT_SIGMOID)
del x

C, S = 96, 64
a = math.radians(30)
theta = torch.tensor([[[math.cos(a), -math.sin(a), 0, 0.2], [math.sin(a), math.cos(a), 0, 0.2], [0, 0, 1.0, 0.2]]]).to(dev)
for D in (64, 16):
    vol = torch.randn(1, D, S, S, C, generator=g).to(dev)
    zs, ys = torch.linspace(-1, 1, D), torch.linspace(-1, 1, S)
    w_, v_, u_ = torch.meshgrid(zs, ys, ys, indexing="ij")
    grid = (torch.stack([u_, v_, w_], -1)[None] + 0.1 * torch.randn(1, D, S, S, 3, generator=g)).contiguous().to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    for _ in range(2):
        ops.l2_flush(flush)
        ops.grid_sample3d(vol, grid=grid, in_layout="cl")
    for _ in range(2):
        ops.l2_flush(flush)
        ops.grid_sample3d(vol, theta=theta, out_size=(D, S, S), in_layout="cl")
torch.cuda.synchronize()
print("done")
