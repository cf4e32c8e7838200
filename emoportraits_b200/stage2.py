"""Stage-2 refinement path (SURVEY.md §8 row a17 / (f) rank 1): drop-in for `notebooks/infer_s2.py:53-387`
InferenceWrapper.forward — `LocalEncoderOld` (`networks/volumetric_avatar/local_encoder_old.py:25-117`) followed by
`Decoder_stage2` / `ImageDecoder_stage2` (`decoder_s2_old.py:18-217, 346-475`), built as in
`models/stage_2/base/volumetric_avatar_two.py:338-444`, all on the same sm_90a kernels as stage 1.  Every residual block is
the stage-1 `nets.ResBlock`; its `nets.Norm` is here the folded BatchNorm, so the blocks carry no statistics.

Default stage-2 configuration (argparse defaults of volumetric_avatar_two.py — the shipped stage-2 args.txt is a
download): norm 'bn' (eval-mode BatchNorm == per-channel affine, folded at load), spectral norm on every conv, no weight
standardisation, encoder 3->128->256->512->512 from output_size_s2 down to 64^2, 1x1 -> 64*16 channels; decoder 1x1
1024->512, 8 ResBlocks @64^2, nearest-x2 ResBlocks 512->256->128->128 up to output_size_s2, feature blocks 128->128->64->32,
BN + ReLU + 1x1 32->3 + Tanh.  The output is an additive residual on the bilinearly resized input.
"""
from __future__ import annotations

import math
import pathlib
from collections import OrderedDict
from dataclasses import dataclass
from typing import Optional

import torch

from . import masks, nets, ops
from .checkpoint import _fill, _sn
from .config import parse_args


@dataclass
class Stage2Config:
    output_size: int = 512        # output_size_s2
    S: int = 64                   # gen_latent_texture_size2
    depth: int = 16               # gen_latent_texture_depth
    C: int = 64                   # gen_latent_texture_channels2
    gen_num_channels: int = 32
    gen_max_channels: int = 512
    enc_channel_mult: float = 4.0  # enc_channel_mult_stage2
    dec_channel_mult: float = 4.0  # dec_channel_mult_stage2
    dec_num_blocks: int = 8        # dec_num_blocks_stage2
    dec_max_channels: int = 512    # dec_max_channels2

    @property
    def enc_channels(self):
        c = int(self.gen_num_channels * self.enc_channel_mult)
        out = [c]
        for _ in range(int(math.log2(self.output_size // self.S))):
            c = min(c * 2, self.gen_max_channels)
            out.append(c)
        return out

    @property
    def dec_width(self):
        nup = int(math.log2(self.output_size // self.S))
        return min(int(self.gen_num_channels * self.dec_channel_mult * 2 ** nup), self.dec_max_channels)

    @property
    def up_channels(self):
        """ImageDecoder_stage2.dec_img_blocks widths (decoder_s2_old.py:374-391): num_up_blocks - 1 halvings"""
        nup = int(math.log2(self.output_size // self.S))
        c = self.dec_width
        out = [c]
        for _ in range(nup - 1):
            c = max(c // 2, self.gen_num_channels)
            out.append(c)
        return out


def stage2_config(args) -> Stage2Config:
    g = lambda k, dflt: getattr(args, k, dflt)
    bad = []
    if g("norm_layer_type", "bn") != "bn":
        bad.append(f"norm_layer_type={g('norm_layer_type', 'bn')} (stage 2 implements the default 'bn')")
    if g("use_ws", False):
        bad.append("use_ws=True")
    if not g("use_sn", True):
        bad.append("use_sn=False")
    for k in ("gen_use_adaconv", "dec_pred_seg", "dec_pred_conf"):
        if g(k, False):
            bad.append(f"{k}=True")
    if bad:
        raise NotImplementedError("stage 2: unsupported configuration: " + "; ".join(bad))
    return Stage2Config(output_size=int(g("output_size_s2", 512)), S=int(g("gen_latent_texture_size2", 64)),
                        depth=int(g("gen_latent_texture_depth", 16)), C=int(g("gen_latent_texture_channels2", 64)),
                        gen_num_channels=int(g("gen_num_channels", 32)), gen_max_channels=int(g("gen_max_channels", 512)),
                        enc_channel_mult=float(g("enc_channel_mult_stage2", 4.0)),
                        dec_channel_mult=float(g("dec_channel_mult_stage2", 4.0)),
                        dec_num_blocks=int(g("dec_num_blocks_stage2", 8)), dec_max_channels=int(g("dec_max_channels2", 512)))


# ------------------------------------------------------------------------------------------------------------------
# checkpoint layout
# ------------------------------------------------------------------------------------------------------------------
def _bn(spec, p, c):
    spec[p + ".weight"] = (c,)
    spec[p + ".bias"] = (c,)
    spec[p + ".running_mean"] = (c,)
    spec[p + ".running_var"] = (c,)
    spec[p + ".num_batches_tracked"] = ()


def _resblock_bn(spec, p, cin, cout, skip):
    _bn(spec, p + ".block_feats.0", cin)
    _sn(spec, p + ".block_feats.2", cout, cin, (3, 3))
    _bn(spec, p + ".block_feats.3", cout)
    _sn(spec, p + ".block.0", cout, cout, (3, 3))
    if skip:
        _sn(spec, p + ".skip.0", cout, cin, (1, 1))


def state_dict_spec_s2(cfg: Stage2Config) -> "OrderedDict[str, tuple]":
    spec: "OrderedDict[str, tuple]" = OrderedDict()
    p = "local_encoder"
    ec = cfg.enc_channels
    s = cfg.output_size
    _sn(spec, f"{p}.from_rgb_{s}px", ec[0], 3, (7, 7), bias=True)
    for i in range(len(ec) - 1):
        _resblock_bn(spec, f"{p}.enc_{i}_block={s}px", ec[i], ec[i + 1], skip=ec[i] != ec[i + 1])
        s //= 2
    _bn(spec, p + ".finale_layers.0", ec[-1])
    _sn(spec, p + ".finale_layers.2", cfg.C * cfg.depth, ec[-1], (1, 1), bias=True)
    p = "decoder"
    w = cfg.dec_width
    _sn(spec, p + ".res_decoder.0", w, cfg.C * cfg.depth, (1, 1))
    for i in range(cfg.dec_num_blocks):
        _resblock_bn(spec, f"{p}.res_decoder.{i + 1}", w, w, skip=False)
    uc = cfg.up_channels
    for i in range(len(uc) - 1):
        _resblock_bn(spec, f"{p}.img_decoder.dec_img_blocks.{i}", uc[i], uc[i + 1], skip=uc[i] != uc[i + 1])
    fc = [uc[-1], 128, 128, 64, 32]  # decoder_s2_old.py:396-423: up block -> 128, then feature blocks 128, 64, 32
    for i in range(4):
        _resblock_bn(spec, f"{p}.img_decoder.dec_img_feat_blocks.{i}", fc[i], fc[i + 1], skip=fc[i] != fc[i + 1])
    _bn(spec, p + ".img_decoder.dec_img_head.0", 32)
    _sn(spec, p + ".img_decoder.dec_img_head.2", 3, 32, (1, 1), bias=True)
    spec["pose_unsqueeze.weight"] = (512 * 16, 512)  # volumetric_avatar_two.py (unused by the inference path)
    return spec


def synthetic_state_dict_s2(cfg: Stage2Config, seed: int = 0):
    """Seeded, well-conditioned weights in the stage-2 checkpoint layout (small gamma in front of the tanh head so the
    additive residual is O(0.1))."""
    return _fill(state_dict_spec_s2(cfg), seed + 1000, small_gamma=(("dec_img_head.0", 0.2),))


# ------------------------------------------------------------------------------------------------------------------
# networks
# ------------------------------------------------------------------------------------------------------------------
def _check_precision(precision):
    if precision not in ("exact", "fast"):
        raise ValueError(f"precision={precision!r}: 'exact' or 'fast'")


class Stage2Model:
    """`model_two.local_encoder` + `model_two.decoder` of notebooks/infer_s2.py:371-372.

    precision="exact" runs every implicit-GEMM convolution on two bf16 operand planes and the 7x7 RGB stem as an fp32 SIMT
    convolution.  precision="fast" runs every convolution on one fp16 plane (ops.H1: one MMA per product), the stem included:
    ops.stem_pack lays its 7 horizontal taps out as channels, so that it becomes a 7x1 implicit GEMM over 32 channels.  The
    error budget is DESIGN.md section 2 (tools/decoder_precision_emulation.py --stage2)."""

    def __init__(self, cfg: Stage2Config, state_dict, device="cuda", precision: str = "exact"):
        _check_precision(precision)
        self.cfg = cfg
        dev = torch.device(device)
        self.device = dev
        sd = state_dict
        self.precision = precision
        self.planes = planes = ops.H1 if precision == "fast" else 2
        p = "local_encoder"
        s = cfg.output_size
        self.stem_w, self.stem_b = nets.stem_weight(sd, f"{p}.from_rgb_{s}px", dev)
        self.stem_h1 = ops.pack_stem_weight(self.stem_w.cpu(), device=dev) if planes == ops.H1 else None
        self.enc = []
        for i in range(len(cfg.enc_channels) - 1):
            self.enc.append(nets.ResBlock(sd, f"{p}.enc_{i}_block={s}px", dev, ws_first=False, planes=planes, pool_fold=True))
            s //= 2
        self.fin_norm = nets.Norm(sd, p + ".finale_layers.0", dev)
        self.fin = nets.ConvW(sd, p + ".finale_layers.2", dev, planes=planes)
        p = "decoder"
        self.inp = nets.ConvW(sd, p + ".res_decoder.0", dev, planes=planes)
        self.res = [nets.ResBlock(sd, f"{p}.res_decoder.{i + 1}", dev, ws_first=False, planes=planes) for i in range(cfg.dec_num_blocks)]
        self.up = [nets.ResBlock(sd, f"{p}.img_decoder.dec_img_blocks.{i}", dev, ws_first=False, planes=planes, subpixel_up=True)
                   for i in range(len(cfg.up_channels) - 1)]
        self.feat = [nets.ResBlock(sd, f"{p}.img_decoder.dec_img_feat_blocks.{i}", dev, ws_first=False, planes=planes, subpixel_up=i == 0)
                     for i in range(4)]
        self.head_norm = nets.Norm(sd, p + ".img_decoder.dec_img_head.0", dev)
        self.head = nets.ConvW(sd, p + ".img_decoder.dec_img_head.2", dev, planes=planes)

    @torch.no_grad()
    def local_encoder(self, x4):
        """x4 (N,1,S,S,4) channels-last (masked, resized) image -> latent (N,1,64,64,C*depth)"""
        return self._encode(ops.stem_pack(x4) if self.stem_h1 is not None else x4)

    def _encode(self, stem_in):
        """local_encoder from the stem's operand: x4 itself (exact) or its stem_pack plane (fast)"""
        if self.stem_h1 is not None:
            x = ops.conv_igemm(stem_in, self.stem_h1, pad=(0, 3, 0), bias=self.stem_b)
        else:
            x = ops.conv_direct(stem_in, self.stem_w, 1, 3, self.stem_b)
        for blk in self.enc:
            x, _ = blk(x, down=(1, 2, 2))
        a = ops.apply(x, **self.fin_norm.apply_args(), act=ops.ACT_RELU, planes=self.planes)
        return ops.conv_igemm(a, self.fin.w, bias=self.fin.b)

    @torch.no_grad()
    def decoder(self, vol):
        """latent channels-last (N,1,64,64,C*depth) -> additive residual (N,3,S,S) NCHW in (-1, 1) (Tanh head)"""
        P = self.planes
        x = ops.conv_igemm(ops.split_bf16(vol, P), self.inp.w)
        for blk in self.res:
            x, _ = blk(x)
        for blk in self.up:
            x, _ = blk(x, up=2)
        x, _ = self.feat[0](x, up=2)
        for blk in self.feat[1:]:
            x, _ = blk(x)
        a = ops.apply(x, **self.head_norm.apply_args(), act=ops.ACT_RELU, planes=P)
        out = ops.conv_igemm(a, self.head.w, bias=self.head.b, act=ops.ACT_TANH, out_nchw=True)
        return out[:, :, 0]

    @torch.no_grad()
    def resize(self, img: torch.Tensor):
        """the bilinear resize (align_corners=False) of img (N,3,h,w) to the output size, both as the encoder's channels-last
        input x4 (N,1,S,S,4), 4th channel 0, and as the NCHW tensor (N,3,S,S) the residual is added to: (x4, resized)"""
        S = self.cfg.output_size
        x4 = ops.resize_bilinear(img.contiguous().float(), (S, S))
        return x4, x4[:, 0, :, :, :3].permute(0, 3, 1, 2).contiguous()

    @torch.no_grad()
    def forward(self, img: torch.Tensor, mask: Optional[torch.Tensor] = None, face_mask: Optional[torch.Tensor] = None):
        """notebooks/infer_s2.py:351-376.  img (N,3,h,w) in [0,1] on device.  Masks default to ones (MODNet / BiSeNet are
        out of scope).  Returns (resized, add, ffhq) NCHW fp32."""
        x4, resized = self.resize(img)
        if mask is not None:
            x4 = (x4 * mask.to(self.device).float().permute(0, 2, 3, 1)[:, None]).contiguous()
        add = self.decoder(self.local_encoder(x4))
        fm = (mask if mask is not None else 1.0)
        if face_mask is not None:
            fm = fm * face_mask.to(self.device).float()
        add = add * fm if not isinstance(fm, float) else add
        ffhq = (resized + add).clamp_(min=0, max=1)
        return resized, add, ffhq

    @torch.no_grad()
    def refine(self, img: torch.Tensor, out: Optional[torch.Tensor] = None, u8: Optional[torch.Tensor] = None, modnet=None,
               face_idt=None, cloth: bool = False, matte: Optional[torch.Tensor] = None, bg: Optional[torch.Tensor] = None,
               threshold: float = 0.3):
        """forward(img)'s ffhq as kernels and the caller's mask networks only, so that a CUDA graph can capture it after a
        stage-1 frame: ops.s2_prepare (the resize and the stem's operand in one pass) -> the encoder and decoder convolutions
        forward runs -> ops.s2_finish (clamp(resized + add, 0, 1) and its uint8 frame in one pass).  img (N,3,h,w) fp32
        contiguous on the device.  out (N,3,S,S) fp32 / u8 (N,S,S,3) uint8: written in place if given.
        matte (N,1,h,w) + bg (3,h,w): img is first composited over bg as video.connect_img_and_bg does (ops.s2_prepare_composite,
        the composited image never in memory).
        modnet (the matting network), face_idt (a masks.FaceParsing or None) and cloth: stage 2's masks, as
        InferenceWrapper.forward computes them with these networks plugged in: the matte of `resized` (masks.modnet_get_mask)
        masks the stem's input (ops.s2_masked_stem), and the matte times the face mask (face_idt.label_masks, kept as uint8;
        the matte alone with cloth or without face_idt) masks the residual (ops.s2_finish_masked).
        Returns (resized, ffhq, u8), bit-identical to forward(x, mask, face_mask)'s resized and ffhq with the same masks, x the
        (composited) image, and to ops.image_to_u8(ffhq)."""
        S, fast = self.cfg.output_size, self.stem_h1 is not None
        if bg is not None:
            resized, stem_in = ops.s2_prepare_composite(img, matte.contiguous().float(), bg, S, None if modnet is not None else fast,
                                                        threshold)
        else:
            resized, stem_in = ops.s2_prepare(img, S, fast=fast)
        if modnet is None:
            add = self.decoder(self._encode(stem_in))
            ffhq, u8 = ops.s2_finish(resized, add, out=out, u8=u8)
            return resized, ffhq, u8
        rmatte = masks.modnet_get_mask(modnet, resized).contiguous()
        face = None if cloth or face_idt is None else face_idt.label_masks(resized)[0]
        # without a composite the prepare pass wrote the unmasked operand: the masked one overwrites it
        stem_in = ops.s2_masked_stem(resized, rmatte, fast, out=stem_in)
        add = self.decoder(self._encode(stem_in))
        ffhq, u8 = ops.s2_finish_masked(resized, add, rmatte, face, out=out, u8=u8)
        return resized, ffhq, u8


class InferenceWrapper(torch.nn.Module):
    """Drop-in for notebooks/infer_s2.py:53 InferenceWrapper (stage 2): same ctor arguments, `forward(img)` returns
    (pil, pil_resized, pil_ffhq, mask).  Reads `project_dir/logs_s2/<experiment_name>/{args.txt, checkpoints/<file>}`."""

    def __init__(self, experiment_name, which_epoch='latest', model_file_name='', use_gpu=True, num_gpus=1,
                 fixed_bounding_box=False, project_dir='./', torch_home='', debug=False, print_model=False,
                 args_overwrite={}, pose_momentum=0.5, experiment_name_s1=None, model_file_name_s1=None, cloth=False,
                 state_dict=None, precision="exact"):
        """precision: "exact" (default: the parity path) or "fast" (every convolution on one fp16 plane, INTEGRATION.md
        "Fast mode"); video.drive_image_with_video runs stage 2 with this setting."""
        super().__init__()
        _check_precision(precision)
        if not use_gpu or not torch.cuda.is_available():
            raise RuntimeError("emoportraits_b200 stage-2 InferenceWrapper needs a CUDA device; there is no CPU path")
        self.cloth = cloth
        args_path = pathlib.Path(project_dir) / 'logs_s2' / experiment_name / 'args.txt'
        self.args = parse_args(args_path)
        self.args.project_dir = project_dir
        for k, v in (args_overwrite or {}).items():
            setattr(self.args, k, v)
        self.cfg = stage2_config(self.args)
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.model_checkpoint_s2 = pathlib.Path(project_dir) / 'logs_s2' / experiment_name / 'checkpoints' / model_file_name
        if state_dict is None:
            state_dict = torch.load(self.model_checkpoint_s2, map_location='cpu')
        self.precision = precision
        self.model_two = Stage2Model(self.cfg, state_dict, self.device, precision=precision)
        # the external mask networks (separate checkouts in the reference: MODNet behind self.modnet, infer_s2.py:134-143, and
        # BiSeNet behind self.face_idt, :71): plug them in as `wrapper.modnet = <module>` /
        # `wrapper.face_idt = masks.FaceParsing(None, net=...)`
        self.modnet = None
        self.face_idt = None

    def check_masks(self) -> None:
        """ValueError unless the plugged-in mask networks are a set forward can use: face_idt needs modnet (the reference's
        residual mask is the matte times the face mask)"""
        if self.face_idt is not None and self.modnet is None:
            raise ValueError("stage 2's face mask multiplies the MODNet matte: plug in wrapper.modnet together with wrapper.face_idt")

    @torch.no_grad()
    def forward(self, img, cloth=False, mask=None, face_mask=None):
        """infer_s2.py:351-376.  img (N,3,h,w) in [0,1].  Returns (pil, pil_resized, pil_ffhq, mask).
        mask (N,1,S,S) / face_mask (N,1,S,S), given by the caller: the stem's input is resized * mask and the residual is
        multiplied by mask * face_mask.  Given neither, with the networks plugged in (modnet, face_idt): the reference's
        masks, computed on the resized image (mask = modnet_get_mask(modnet, resized), face_mask = face_idt.forward(resized)[0],
        no face mask with cloth=True), and the fourth output is the matte of img clamped to [0, 1].  Without networks and
        masks stage 2 runs unmasked and the fourth output is ones."""
        from PIL import Image

        img = img.to(self.device).float()
        pred_mask = None
        if mask is None and face_mask is None and self.modnet is not None:
            self.check_masks()
            pred_mask = masks.modnet_get_mask(self.modnet, img)                             # :356
            _, resized = self.model_two.resize(img)                                         # :360
            mask = masks.modnet_get_mask(self.modnet, resized)                              # :361
            if self.face_idt is not None:
                face_mask = self.face_idt.forward(resized)[0]                               # :362
        if self.cloth:
            face_mask = None  # infer_s2.py:365-368: with cloth=True the refinement is not restricted to the face region
        resized, add, ffhq = self.model_two.forward(img, mask, face_mask)
        to_pil = lambda t: [Image.fromarray(h) for h in ops.image_to_u8(t.detach().contiguous().float()).cpu().numpy()]
        m = pred_mask if pred_mask is not None else mask if mask is not None else torch.ones_like(img[:, :1])
        return to_pil(img), to_pil(resized), to_pil(ffhq), m.detach().cpu().clamp(0, 1)
