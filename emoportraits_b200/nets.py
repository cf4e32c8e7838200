"""Network assembly of the volumetric-avatar hot path on top of the C-ABI ops.

Each class mirrors one reference module (same name, same checkpoint prefix, same call order) but holds
pre-folded, kernel-native weights and launches only emoportraits_b200 kernels:

    LocalEncoder      networks/volumetric_avatar/local_encoder.py:26-125
    ResNet (18/50)    torchvision resnet as wrapped by identity_embedder.py:12-89, expression_embedder.py:343-478,
                      head_pose_regressor.py:11-31
    WarpGenerator     networks/volumetric_avatar/warp_generator_resnet.py:11-181
    VolumeSource      vpn_resblocks.py:22-49 -> resblocks_3d.py:9-62
    Unet3D            networks/volumetric_avatar/unet_3d.py:18-290
    Decoder           networks/volumetric_avatar/decoder.py:20-410
    ResBlock          networks/volumetric_avatar/utils.py:661-788

Data flowing between layers is a channels-last fp32 tensor (N, D, H, W, C) plus the GroupNorm statistics of that
tensor (double (N,32,2)), produced by the epilogue of whichever kernel wrote it.
"""
from __future__ import annotations

import math

import torch

from . import ops
from .checkpoint import fold_conv
from .config import HotPathConfig

G = 32


class ConvW:
    """Packed conv weight (+ bias) resident on the device."""

    def __init__(self, sd, p, dev, ws=False, in_perm=None, out_perm=None, planes=2):
        w, b = fold_conv(sd, p, ws=ws)
        if out_perm is not None:
            w = w[out_perm]
            b = b[out_perm] if b is not None else None
        self.w = ops.pack_conv_weight(w, device=dev, in_perm=in_perm, planes=planes)
        self.b = b.to(dev).contiguous() if b is not None else None
        self.cout = w.shape[0]


class Norm:
    """GroupNorm(32), or eval-mode BatchNorm (recognised by its `running_mean`) folded to the per-channel y = x*A + B."""

    def __init__(self, sd, p, dev):
        self.gamma = sd[p + ".weight"].detach().float().to(dev).contiguous()
        self.beta = sd[p + ".bias"].detach().float().to(dev).contiguous()
        self.needs_stats = (p + ".running_mean") not in sd
        if not self.needs_stats:
            g, b = sd[p + ".weight"].float(), sd[p + ".bias"].float()
            m, v = sd[p + ".running_mean"].float(), sd[p + ".running_var"].float()
            A = g / torch.sqrt(v + 1e-5)
            self.A = A[None].to(dev).contiguous()
            self.B = (b - m * A)[None].to(dev).contiguous()

    def affine(self, stats, count):
        if not self.needs_stats:
            return self.A, self.B
        return ops.gn_finalize(stats, count, self.gamma, self.beta)

    def gn(self, stats, count, ada=None):
        """arguments of the GroupNorm finalisation fused into ops.apply"""
        d = dict(stats=stats, count=count, gamma=self.gamma, beta=self.beta)
        if ada is not None:
            d.update(ada_w=ada[0], ada_b=ada[1])
        return d

    def apply_args(self, stats=None, count=None, ada=None):
        """keyword arguments of ops.apply (or of a conv `post=`) that normalise a tensor whose statistics are `stats`"""
        if not self.needs_stats:
            return dict(A=self.A, B=self.B, per_sample=False)
        return dict(gn=self.gn(stats, count, ada))


def _count(x):
    """elements per (sample, group) of a channels-last tensor"""
    return x.numel() / x.shape[0] / G


def stem_weight(sd, p, dev):
    """7x7 RGB stem conv -> ops.conv_direct operands: weight (7, 7, 4, Cout) with a zero 4th input channel, bias"""
    w, b = fold_conv(sd, p)
    wc = torch.zeros(7, 7, 4, w.shape[0])
    wc[:, :, :3] = w.permute(2, 3, 1, 0)
    return wc.to(dev).contiguous(), (b.to(dev).contiguous() if b is not None else None)


class ResBlock:
    """utils.py:661-788: [nearest up] -> norm -> relu -> conv -> norm -> relu -> conv [-> avgpool]; skip = [up] -> [1x1] -> [pool].
    The norms are GroupNorm (stage 1) or eval-mode BatchNorm (stage 2); only GroupNorm needs statistics."""

    def __init__(self, sd, p, dev, ws_first=True, planes=2, subpixel_up=False, pool_fold=False):
        self.planes = planes
        self.n1 = Norm(sd, p + ".block_feats.0", dev)
        self.c1 = ConvW(sd, p + ".block_feats.2", dev, ws=ws_first, planes=planes)
        # sub-pixel form of `nearest x2 -> norm -> relu -> 3x3 conv` for blocks called with up=2 (ops.pack_upconv_weight):
        # the conv then reads the LOW-resolution planes (4/9 of the MMAs, no upsampled operand; measured round 2: 229 -> 244
        # frames/s).  Shapes the sub-pixel kernel does not take (Cout % 32, Cin % 64, odd pixel-tile count) use the plain form.
        # Two bf16 planes or one fp16 plane (ops.H1).
        self.c1_ps = None
        if subpixel_up and planes in (2, ops.H1):
            w, _ = fold_conv(sd, p + ".block_feats.2", ws=ws_first)
            if tuple(w.shape[2:]) == (3, 3) and w.shape[0] % 32 == 0 and w.shape[1] % 64 == 0:
                self.c1_ps = ops.pack_upconv_weight(w, device=dev, planes=planes)
        self.n2 = Norm(sd, p + ".block_feats.3", dev)
        self.c2 = ConvW(sd, p + ".block.0", dev, planes=planes)
        self.skip = ConvW(sd, p + ".skip.0", dev, planes=planes) if (p + ".skip.0.weight_orig") in sd else None
        # `conv -> avgpool (1,2,2)` of down-sampling blocks folded into one 4x4 stride-2 conv (ops.fold_poolconv_weight):
        # 16 taps per pooled output instead of 36 and no full-resolution conv output (stage-2 @1024^2: 37.5 -> 44.4 images/s
        # together with the sub-pixel form).
        self.c2_pool = None
        if pool_fold:
            w, _ = fold_conv(sd, p + ".block.0")
            if tuple(w.shape[2:]) == (3, 3):
                self.c2_pool = ops.pack_conv_weight(ops.fold_poolconv_weight(w), device=dev, planes=planes)

    def __call__(self, x, sx=None, up=1, down=None, ada=None, want_stats=True):
        """x and its statistics sx (None for BatchNorm) -> (out, statistics of out: None for BatchNorm or want_stats=False)"""
        dev = x.device
        N = x.shape[0]
        st1 = ops.new_stats(N, G, dev) if self.n2.needs_stats else None
        subpixel = up == 2 and self.c1_ps is not None and x.shape[1] == 1 and (x.shape[2] * x.shape[3]) % 256 == 0
        a = ops.apply(x, **self.n1.apply_args(sx, _count(x), ada[0] if ada else None), act=ops.ACT_RELU, up=1 if subpixel else up,
                      planes=self.planes)
        if subpixel:
            y = ops.conv_igemm(a, self.c1_ps, bias=self.c1.b, stats=st1, upconv=True)
            b = ops.apply(y, **self.n2.apply_args(st1, _count(y), ada[1] if ada else None), act=ops.ACT_RELU, planes=self.planes)
        else:
            # conv -> norm -> relu: the second norm's pass is the convolution's post-op (one launch for the small split-K layers)
            cnt = a.shape[1] * a.shape[2] * a.shape[3] * self.c1.cout / G
            b = ops.conv_igemm(a, self.c1.w, bias=self.c1.b, stats=st1,
                               post=dict(**self.n2.apply_args(st1, cnt, ada[1] if ada else None), act=ops.ACT_RELU, planes=self.planes))
        # skip path: the 1x1 conv commutes with nearest-upsampling and with average pooling, so it runs at the smaller size
        s = ops.avgpool(x, down) if down else x
        if self.skip is not None:
            s = ops.conv_igemm(ops.split_bf16(s, self.planes), self.skip.w, bias=self.skip.b)
        st2 = ops.new_stats(N, G, dev) if (want_stats and self.n2.needs_stats) else None
        if down and self.c2_pool is not None and tuple(down) == (1, 2, 2) and b.shape[2] % 2 == 0 and b.shape[3] % 2 == 0:
            out = ops.conv_igemm(b, self.c2_pool, stride=(1, 2, 2), pad=(0, 1, 1), bias=self.c2.b, residual=s, stats=st2)
        elif down:
            full = ops.conv_igemm(b, self.c2.w, bias=self.c2.b)
            out = ops.avgpool(full, down, add=s, stats=st2)
        else:
            out = ops.conv_igemm(b, self.c2.w, bias=self.c2.b, residual=s, res_shift=1 if up == 2 else 0, stats=st2)
        return out, st2


# ------------------------------------------------------------------------------------------------------------------
class LocalEncoder:
    def __init__(self, sd, cfg: HotPathConfig, dev, planes=2):
        self.planes = planes
        p = "local_encoder_nw"
        s = cfg.image_size
        self.stem_w, self.stem_b = stem_weight(sd, f"{p}.from_rgb_{s}px", dev)
        # one fp16 plane: the stem runs on the tensor cores as a 7x1 implicit GEMM over ops.stem_pack's 32 channels
        self.stem_h1 = ops.pack_stem_weight(self.stem_w.cpu(), device=dev) if planes == ops.H1 else None
        self.blocks = []
        for i in range(len(cfg.enc_channels) - 1):
            self.blocks.append(ResBlock(sd, f"{p}.enc_{i}_block={s}px", dev, planes=planes, pool_fold=True))
            s //= 2
        self.fin_norm = Norm(sd, p + ".finale_layers.0", dev)
        # output channel o = c*D + d in the reference (infer.py:485 view(1,c,d,s,s)); emit d*C + c so the map is (h,w,d,c)
        C, D = cfg.C, cfg.D
        operm = torch.tensor([(k % C) * D + (k // C) for k in range(C * D)])
        self.fin = ConvW(sd, p + ".finale_layers.2", dev, ws=True, out_perm=operm, planes=planes)
        self.cfg = cfg

    def __call__(self, img_nchw):
        """img (1,3,H,W) fp32 -> latent volume channels-last (1,D,S,S,C) fp32 + its GN stats."""
        cfg = self.cfg
        x4 = ops.resize_bilinear(img_nchw, img_nchw.shape[-2:])  # same-size bilinear == exact NCHW -> NHWC4 repack
        st = ops.new_stats(1, G, x4.device)
        if self.stem_h1 is not None:
            x = ops.conv_igemm(ops.stem_pack(x4), self.stem_h1, pad=(0, 3, 0), bias=self.stem_b, stats=st)
        else:
            x = ops.conv_direct(x4, self.stem_w, 1, 3, self.stem_b, stats=st)
        for blk in self.blocks:
            x, st = blk(x, st, down=(1, 2, 2))
        a = ops.apply(x, gn=self.fin_norm.gn(st, _count(x)), act=ops.ACT_RELU, planes=self.planes)
        y = ops.conv_igemm(a, self.fin.w, bias=self.fin.b)  # (1,1,S,S,D*C) == (h,w,d,c)
        vol = y.view(1, cfg.S, cfg.S, cfg.D, cfg.C).permute(0, 3, 1, 2, 4).contiguous()  # -> (1,D,S,S,C)
        return vol


# ------------------------------------------------------------------------------------------------------------------
class ResNet:
    """torchvision resnet18 / resnet50 trunk (conv1..layer4) on channels-last tensors; the norms are eval-mode BatchNorm or
    GroupNorm(32) (replace_bn_to_gn, utils.py:1020)."""

    def __init__(self, sd, p, dev, gn: bool, planes=2):
        self.gn = gn
        self.planes = planes
        self.stem_w, self.stem_b = stem_weight(sd, p + ".conv1", dev)
        self.bn1 = Norm(sd, p + ".bn1", dev)
        self.blocks = []
        for li in range(1, 5):
            bi = 0
            while f"{p}.layer{li}.{bi}.bn1.weight" in sd:
                q = f"{p}.layer{li}.{bi}"
                blk = dict(stride=2 if (li > 1 and bi == 0) else 1, bottleneck=(q + ".bn3.weight") in sd)
                blk["c1"] = ConvW(sd, q + ".conv1", dev, planes=planes)
                blk["n1"] = Norm(sd, q + ".bn1", dev)
                blk["c2"] = ConvW(sd, q + ".conv2", dev, ws=gn, planes=planes)
                blk["n2"] = Norm(sd, q + ".bn2", dev)
                if blk["bottleneck"]:
                    blk["c3"] = ConvW(sd, q + ".conv3", dev, ws=gn, planes=planes)
                    blk["n3"] = Norm(sd, q + ".bn3", dev)
                if (q + ".downsample.1.weight") in sd:
                    blk["cd"] = ConvW(sd, q + ".downsample.0", dev, planes=planes)
                    blk["nd"] = Norm(sd, q + ".downsample.1", dev)
                self.blocks.append(blk)
                bi += 1

    def _conv(self, a, cw, stride=1):
        st = ops.new_stats(a.shape[0], G, a.hi.device) if self.gn else None
        y = ops.conv_igemm(a, cw.w, stride=(1, stride, stride), bias=cw.b, stats=st)
        return y, st

    def _conv_norm(self, a, cw, norm, stride=1, **kw):
        """conv -> norm (-> + residual) -> relu as one call: the norm pass is the convolution's post-op (emo_conv_desc.post; the
        ResNet layers are small split-K layers, so this is one finalize launch instead of finalize + apply).  eval-BatchNorm is
        a per-channel affine; GroupNorm is finalised from the convolution's own statistics."""
        kw.setdefault("planes", self.planes)
        N, _, Hi, Wi, _ = a.shape
        st = ops.new_stats(N, G, a.hi.device) if norm.needs_stats else None
        k = cw.w.k[1]
        Ho, Wo = (Hi + 2 * (k // 2) - k) // stride + 1, (Wi + 2 * (k // 2) - k) // stride + 1
        return ops.conv_igemm(a, cw.w, stride=(1, stride, stride), bias=cw.b, stats=st,
                              post=dict(**norm.apply_args(st, Ho * Wo * cw.cout / G), **kw))

    def __call__(self, x4):
        """x4 (N,1,H,W,4) normalised image, channels-last padded -> (N,1,H/32,W/32,C) fp32."""
        N, dev = x4.shape[0], x4.device
        st = ops.new_stats(N, G, dev) if self.gn else None
        y = ops.conv_direct(x4, self.stem_w, 2, 3, self.stem_b, stats=st)
        y = ops.apply(y, **self.bn1.apply_args(st, _count(y)), act=ops.ACT_RELU, want_f32=True, want_split=False)
        x = ops.maxpool2d_3x3s2(y)
        xs = ops.split_bf16(x, self.planes)
        relu = dict(act=ops.ACT_RELU)
        for blk in self.blocks:
            s = blk["stride"]
            if blk["bottleneck"]:
                a = self._conv_norm(xs, blk["c1"], blk["n1"], **relu)
                a = self._conv_norm(a, blk["c2"], blk["n2"], s, **relu)
                last_c, last_n, last_s = blk["c3"], blk["n3"], 1
            else:
                a = self._conv_norm(xs, blk["c1"], blk["n1"], s, **relu)
                last_c, last_n, last_s = blk["c2"], blk["n2"], 1
            if "cd" in blk:
                r, std = self._conv(xs, blk["cd"], s)
                A2, B2 = blk["nd"].affine(std, _count(r))
                # residual affine is per-channel in the kernel; with GN and N == 1 the per-sample row is that vector
                assert not last_n.needs_stats or N == 1, "GN ResNet path runs one image at a time"
                x, xs = self._conv_norm(a, last_c, last_n, last_s, res=r, A2=A2, B2=B2, want_f32=True, want_split=True, **relu)
            else:
                x, xs = self._conv_norm(a, last_c, last_n, last_s, res=x, want_f32=True, want_split=True, **relu)
        return x, xs


def _norm_buffers(sd, p, dev):
    """input normalisation of an embedder: its `mean` / `std` buffers from the checkpoint (identity_embedder.py:21-22,
    expression_embedder.py:352-353 register the ImageNet statistics), the ImageNet constants if the checkpoint has none"""
    mean = sd[p + ".mean"].detach().float().reshape(-1) if (p + ".mean") in sd else torch.tensor([0.485, 0.456, 0.406])
    std = sd[p + ".std"].detach().float().reshape(-1) if (p + ".std") in sd else torch.tensor([0.229, 0.224, 0.225])
    return mean.to(dev).contiguous(), std.to(dev).contiguous()


class HeadPoseRegressor:
    """head_pose_regressor.py:11-31 — resnet18(num_classes=9), BatchNorm, its own checkpoint."""

    def __init__(self, hsd, dev, planes=2):
        sd = {"r." + k: v for k, v in hsd.items()}
        self.net = ResNet(sd, "r", dev, gn=False, planes=planes)
        self.fc_w = sd["r.fc.weight"].float().to(dev).contiguous()
        self.fc_b = sd["r.fc.bias"].float().to(dev).contiguous()

    def __call__(self, img_nchw):
        x4 = ops.resize_bilinear(img_nchw, (128, 128))
        f, _ = self.net(x4)
        return ops.linear(ops.global_avgpool(f), self.fc_w, self.fc_b)  # (N, 9) = scale, rotation, translation


class ExpressionEmbed:
    """expression_embedder.py:132-253 (inference branch) + ResNetWrapper :441-478."""

    def __init__(self, sd, cfg: HotPathConfig, dev, planes=2):
        p = "expression_embedder_nw.net_face"
        self.net = ResNet(sd, p + ".net", dev, gn=True, planes=planes)
        self.fc = ConvW(sd, p + ".net.fc", dev, planes=planes)
        w, _ = fold_conv(sd, p + ".pose_head")  # (E, E*16), input index c*16 + s (torch.flatten of NCHW)
        E = cfg.expr_channels
        self.head_w = w.view(E, E, 16).permute(0, 2, 1).reshape(E, 16 * E).to(dev).contiguous()  # -> index s*E + c
        self.mean, self.std = _norm_buffers(sd, p, dev)
        self.grid = cfg.exp_image_size // 2

    def __call__(self, img_nchw, align2d, want_aligned=False):
        res = ops.grid_sample2d_affine(img_nchw, align2d, (self.grid, self.grid), self.mean, self.std, want_nchw=want_aligned)
        x4, aligned = (res if want_aligned else (res, None))
        _, fs = self.net(x4)
        y = ops.conv_igemm(fs, self.fc.w, bias=self.fc.b)  # (N,1,4,4,E); AdaptiveAvgPool2d(4) is the identity here
        N = y.shape[0]
        assert y.shape[2] == 4 and y.shape[3] == 4, "exp_image_size other than 256 needs a real adaptive pool"
        emb = ops.linear(y.view(N, -1), self.head_w)
        return emb, aligned


class IdtEmbed:
    """identity_embedder.py:59-89: bilinear -> 256, normalise, resnet50 (GN), fc 1x1 conv, AdaptiveAvgPool2d(4)."""

    def __init__(self, sd, cfg: HotPathConfig, dev, planes=2):
        p = "idt_embedder_nw"
        self.net = ResNet(sd, p + ".net", dev, gn=True, planes=planes)
        self.fc = ConvW(sd, p + ".net.fc", dev, planes=planes)
        self.mean, self.std = _norm_buffers(sd, p, dev)
        self.size = cfg.idt_image_size

    def __call__(self, img_nchw):
        x4 = ops.resize_bilinear(img_nchw, (self.size, self.size), self.mean, self.std)
        _, fs = self.net(x4)
        y = ops.conv_igemm(fs, self.fc.w, bias=self.fc.b)  # (1,1,8,8,512)
        y = ops.avgpool(y, (1, y.shape[2] // 4, y.shape[3] // 4)) if y.shape[2] != 4 else y
        # reference layout of idt_embed is NCHW (1,512,4,4); keep that for the wrapper API and predict_embed
        return y[:, 0].permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------------------------
class PredictEmbed:
    """va.py:813-885 (gen_pred_mixing True, cat_em False): 'orig' = conv1x1((pose_unsqueeze(pose) + idt) * 0.5)."""

    def __init__(self, sd, cfg: HotPathConfig, dev):
        self.w_unsq = sd["pose_unsqueeze_nw.weight"].detach().float().to(dev).contiguous()
        w, _ = fold_conv(sd, "warp_embed_head_orig_nw")
        self.w_head = w.reshape(w.shape[0], w.shape[1]).to(dev).contiguous()
        self.Cm = cfg.gen_max_channels
        self.es2 = cfg.embed_size ** 2

    def __call__(self, pose_embed, idt_nchw):
        """pose (1,E), idt (1,512,4,4) NCHW -> E 'orig' (1,512,16) [c][s] contiguous."""
        h = ops.linear(pose_embed, self.w_unsq, add=idt_nchw.reshape(1, -1), scale=0.5)  # (1, 512*16) index c*16+s
        E = torch.empty((1, self.Cm, self.es2), dtype=torch.float32, device=h.device)
        ops.linear(h, self.w_head, x_strides=(1, self.es2), M=self.es2, K=self.Cm, out=E, out_strides=(1, self.es2))
        return E


class WarpGenerator:
    def __init__(self, sd, p, cfg: HotPathConfig, dev, planes=2):
        self.cfg = cfg
        self.planes = planes
        ch = cfg.warp_channels
        self.ch = ch
        isz = cfg.embed_size
        w, _ = fold_conv(sd, p + ".first_conv")
        w = w.reshape(w.shape[0], w.shape[1])  # (ch0*isz, 512); out index o = c*isz + d (view(b,-1,isz,isz,isz))
        self.first_w = [w[d::isz].to(dev).contiguous() for d in range(isz)]  # per depth slice: rows c -> o = c*isz+d
        self.blocks = [ResBlock(sd, f"{p}.blocks_3d.{i}", dev, ws_first=True, planes=planes) for i in range(len(ch) - 1)]
        self.pu, self.pvT = [], []
        j = 0
        while f"{p}.projector.u.{j}" in sd:
            self.pu.append(sd[f"{p}.projector.u.{j}"].detach().float().to(dev).contiguous())
            self.pvT.append(sd[f"{p}.projector.v.{j}"].detach().float().t().to(dev).contiguous())  # (2,16)
            j += 1
        self.pre_head = Norm(sd, p + ".pre_head.0", dev)
        self.head = ConvW(sd, p + ".head.0.0", dev, planes=planes)
        idg = sd[p + ".identity_grid"].detach().float()  # (1,3,D,S,S) -> (D,S,S,3)
        self.idg = idg[0].permute(1, 2, 3, 0).contiguous().to(dev)
        self._prepare_ada()

    def _prepare_ada(self):
        """ProjectorNorm (utils.py:1140-1151) for ALL AdaptiveGroupNorm layers in two launches instead of two per layer:
        (u_j . E . v_j) = u_j . (E . v_j), so  EV = E . [v_0 | v_1 | ...]  (512 x 2L, one small GEMM) and then
        OUT = [u_0; u_1; ...] . EV + [gamma_j, beta_j in layer j's two columns]  (sum C_j x 2L, one GEMM: every layer reads only
        its own column pair; the other columns are wasted flops of a 8 MFLOP product).  OUT is written transposed, so that
        (gamma + dgamma, beta + dbeta) of layer j are two contiguous rows slices."""
        norms = []
        for blk in self.blocks:
            norms += [blk.n1, blk.n2]
        L = len(self.pu)
        assert L == len(norms)
        dev = self.pu[0].device
        self.ada_rows = [0]
        for u in self.pu:
            self.ada_rows.append(self.ada_rows[-1] + u.shape[0])
        Ctot = self.ada_rows[-1]
        self.ada_U = torch.cat(self.pu, 0).contiguous()                                            # (Ctot, 512)
        self.ada_V = torch.cat(self.pvT, 0).contiguous()                                           # (2L, 16): row 2j+i = v_j[:, i]
        add = torch.zeros((2 * L, Ctot), dtype=torch.float32, device=dev)
        for j, nrm in enumerate(norms):
            add[2 * j, self.ada_rows[j]:self.ada_rows[j + 1]] = nrm.gamma
            add[2 * j + 1, self.ada_rows[j]:self.ada_rows[j + 1]] = nrm.beta
        self.ada_add = add.contiguous()
        self.ada_L = L

    def _ada_all(self, E):
        """E (512,16) -> list over layers of (ada_w (1,C_j), ada_b (1,C_j))"""
        L, Ctot, K = self.ada_L, self.ada_rows[-1], E.shape[0]
        EVt = torch.empty((2 * L, K), dtype=torch.float32, device=E.device)                        # EVt[q][k] = sum_s E[k][s] V[q][s]
        ops.linear(E, self.ada_V, x_strides=(16, 1), M=K, K=16, out=EVt, out_strides=(1, K))
        out = torch.empty((2 * L, Ctot), dtype=torch.float32, device=E.device)                     # out[q][c] = sum_k U[c][k] EVt[q][k] + add[q][c]
        ops.linear(self.ada_U, EVt, add=self.ada_add, x_strides=(K, 1), M=Ctot, K=K, out=out, out_strides=(1, Ctot))
        return [(out[2 * j:2 * j + 1, self.ada_rows[j]:self.ada_rows[j + 1]], out[2 * j + 1:2 * j + 2, self.ada_rows[j]:self.ada_rows[j + 1]])
                for j in range(L)]

    def __call__(self, E):
        """E (1,512,16) -> warp (1,D,S,S,3) fp32 channels-last == the (b,D,H,W,3) grid of the reference."""
        cfg = self.cfg
        assert E.shape[0] == 1, "per-frame call (batch the frames over ranks/streams, not here)"
        dev = E.device
        isz = cfg.embed_size
        Em = E[0]
        x = torch.empty((1, isz, isz, isz, self.ch[0]), dtype=torch.float32, device=dev)
        for d in range(isz):  # first_conv 1x1 on the 4x4 map, written straight into the (d,h,w,c) volume
            ops.linear(Em, self.first_w[d], x_strides=(1, isz * isz), M=isz * isz, K=Em.shape[0], out=x[0, d],
                       out_strides=(self.ch[0], 1))
        size = [isz, isz, isz]
        ndr = int(math.log2(cfg.S // isz))
        nblk = len(self.blocks)
        st = None
        adas = self._ada_all(Em)
        for i in range(1, nblk + 1):
            size[1] *= 2
            size[2] *= 2
            depth_new = min(cfg.D * 2 ** (ndr - i), size[1]) if i < ndr else cfg.D
            up_depth, down_depth = depth_new > size[0], depth_new < size[0]
            size[0] = depth_new
            st = ops.new_stats(1, G, dev)
            x = ops.upsample_trilinear(x, (2, 2, 2) if up_depth else (1, 2, 2), stats=st)
            blk = self.blocks[i - 1]
            ada = (adas[2 * (i - 1)], adas[2 * (i - 1) + 1])
            x, st = blk(x, st, ada=ada, want_stats=not down_depth)
            if down_depth:
                st = ops.new_stats(1, G, dev)
                x = ops.avgpool(x, (2, 1, 1), stats=st)
        a = ops.apply(x, gn=self.pre_head.gn(st, _count(x)), act=ops.ACT_RELU, planes=self.planes)
        return ops.conv_igemm(a, self.head.w, bias=self.head.b, act=ops.ACT_TANH, post_add=self.idg)


class VolumeSource:
    def __init__(self, sd, cfg: HotPathConfig, dev, planes=2):
        self.blocks = [ResBlock(sd, f"volume_source_nw.net.net.{i}", dev, ws_first=False, planes=planes)
                       for i in range(cfg.source_volume_num_blocks)]

    def __call__(self, vol):
        st = ops.gn_stats(vol, G)
        for i, blk in enumerate(self.blocks):
            vol, st = blk(vol, st, want_stats=i < len(self.blocks) - 1)
        return vol


class Unet3D:
    def __init__(self, sd, cfg: HotPathConfig, dev, planes=2):
        p = "volume_process_nw"
        self.cfg = cfg
        self.planes = planes
        nb = len(cfg.unet_channels) - 1
        self.nb = nb
        self.down = [ResBlock(sd, f"{p}.blocks_3d_down.{i}", dev, ws_first=False, planes=planes) for i in range(nb)]
        self.up = [ResBlock(sd, f"{p}.blocks_3d_up.{i}", dev, ws_first=False, planes=planes) for i in range(nb)]
        self.skipb = [ResBlock(sd, f"{p}.skip_blocks_3d_up.{i}", dev, ws_first=False, planes=planes) for i in range(nb)]
        it = sd[p + ".input_tensor"].detach().float()  # (1,C,8,8,8)
        self.seed = it.permute(0, 2, 3, 4, 1).contiguous().to(dev)
        self.head_norm = Norm(sd, p + ".head.0", dev)
        self.head = ConvW(sd, p + ".head.2", dev, planes=planes)

    def __call__(self, vol):
        cfg, dev, nb = self.cfg, vol.device, self.nb
        x = vol
        feats = []
        size = [cfg.D, vol.shape[2], vol.shape[3]]
        st = None
        for i in range(nb):
            kind = "none"
            if i < nb - 1:
                size[1] //= 2
                size[2] //= 2
                depth_new = min(size[0] * 2, size[1])
                kind = "up" if depth_new > size[0] else ("down" if depth_new < size[0] else "none")
                size[0] = depth_new
            if kind == "up":
                st = ops.new_stats(1, G, dev)
                x = ops.upsample_trilinear(x, (2, 1, 1), stats=st)
            elif st is None:
                st = ops.gn_stats(x, G)
            x, st_out = self.down[i](x, st)
            feats.append((x, st_out))
            if i < nb - 1:
                st = ops.new_stats(1, G, dev)
                x = ops.avgpool(x, (2, 2, 2) if kind == "down" else (1, 2, 2), stats=st)
        feats = feats[::-1]
        x = self.seed
        size = [x.shape[1], x.shape[2], x.shape[3]]
        st = None
        for i in range(1, nb + 1):
            size[1] *= 2
            size[2] *= 2
            depth_new = min(cfg.D * 2 ** (nb - i), size[1])
            kind = "up" if depth_new > size[0] else ("down" if depth_new < size[0] else "none")
            size[0] = depth_new
            f, fst = feats[i - 1]
            skip, _ = self.skipb[i - 1](f, fst, want_stats=False)
            st = ops.new_stats(1, G, dev)
            x = ops.upsample_trilinear(x, (2, 2, 2) if kind == "up" else (1, 2, 2), add=skip, stats=st)
            x, st = self.up[i - 1](x, st, want_stats=kind != "down")
            if kind == "down":
                st = ops.new_stats(1, G, dev)
                x = ops.avgpool(x, (2, 1, 1), stats=st)
        a = ops.apply(x, gn=self.head_norm.gn(st, _count(x)), act=ops.ACT_RELU, planes=self.planes)
        return ops.conv_igemm(a, self.head.w, bias=self.head.b)


class Decoder:
    def __init__(self, sd, cfg: HotPathConfig, dev, planes=2):
        self.planes = planes
        p = "decoder_nw"
        C, D = cfg.C, cfg.D
        # the warped volume arrives as (h, w, d, c): channel k' = d*C + c  <->  reference channel c*D + d (infer.py:627)
        iperm = torch.tensor([(k % C) * D + (k // C) for k in range(C * D)])
        self.inp = ConvW(sd, p + ".res_decoder.0", dev, in_perm=iperm, planes=planes)
        self.res = [ResBlock(sd, f"{p}.res_decoder.{i + 1}", dev, planes=planes) for i in range(cfg.dec_num_blocks)]
        self.img = []
        j = 0
        while f"{p}.img_decoder.dec_img_blocks.{j}.block.0.weight_orig" in sd:
            self.img.append(ResBlock(sd, f"{p}.img_decoder.dec_img_blocks.{j}", dev, planes=planes,
                                     subpixel_up=(j % cfg.im_dec_lrs == 0)))
            j += 1
        self.lrs = cfg.im_dec_lrs
        self.head_norm = Norm(sd, p + ".img_decoder.dec_img_head.0", dev)
        # dec_img_head (decoder.py:398-410): norm -> ReLU -> 1x1 Conv2d_ws -> sigmoid runs as ONE exact-fp32 pass (ops.gn_head)
        hw, hb = fold_conv(sd, p + ".img_decoder.dec_img_head.2", ws=True)
        assert tuple(hw.shape[2:]) == (1, 1) and hw.shape[0] <= 4, hw.shape
        self.head_w = hw.reshape(hw.shape[0], hw.shape[1]).float().to(dev).contiguous()
        self.head_b = hb.float().to(dev).contiguous() if hb is not None else None

    def __call__(self, feat: "ops.Split", want_logits: bool = False):
        """feat: Split (N,1,S,S,C*D) in (h,w,d,c) order -> img (N,3,H,W) fp32 NCHW, feat_2d, img_feat."""
        N, dev = feat.shape[0], feat.hi.device
        st = ops.new_stats(N, G, dev)
        x = ops.conv_igemm(feat, self.inp.w, stats=st)
        for blk in self.res:
            x, st = blk(x, st)
        feat2d = x
        for j, blk in enumerate(self.img):
            x, st = blk(x, st, up=2 if (j % self.lrs == 0) else 1)
        img = ops.gn_head(x, self.head_norm.gn(st, _count(x)), self.head_w, self.head_b,
                          act_out=ops.ACT_NONE if want_logits else ops.ACT_SIGMOID)
        return img[:, :, 0], feat2d, x
