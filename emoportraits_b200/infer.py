"""Drop-in for the reference's stage-1 inference API: `notebooks/infer.py:62-647` InferenceWrapper.

Same constructor and `forward` signature, same `args.txt` / checkpoint layout (`project_dir/folder/experiment_name/
{args.txt, checkpoints/<model_file_name>}`), same cached source state on `self`, same return value
`(list[PIL.Image], img Tensor (B,3,H,W) fp32 on device)`.  The hot path underneath is emoportraits_b200's sm_90a
kernels; there is no torch/CPU fallback — without an H100 and the built libemoport.so this module raises.

Out of scope here (SURVEY.md §2 rows 8, §8f rank 3): the external face detector (`crop=True` raises) and the WEIGHTS / model
code of the external mask networks (MODNet, BiSeNet: separate checkouts, not in the reference tree).  The processing the
reference does around them is here (`masks.py`, csrc/masks.cu): plug the networks in with `wrapper.face_idt =
masks.FaceParsing(None, net=...)` / `wrapper.modnet = ...`; without them the source mask is `source_mask` or all ones (what the
stubbed reference oracle uses too) and `modnet_mask=True` raises.
"""
from __future__ import annotations

import copy
import pathlib
from collections import OrderedDict
from types import SimpleNamespace
from typing import Optional

import numpy as np
import torch

from . import nets, ops
from .config import HotPathConfig, hot_path_config, parse_args
from .dist import check_identity, new_identity, source_state_shapes


class Model:
    """Inference-only counterpart of models/stage_1/volumetric_avatar/va.py:39 Model (attribute names kept)."""

    # Operand planes per network (ops.conv_igemm): 2 = two bf16 planes, 3 MMAs per product, ~2^-16 relative (decoder: isolated
    # stage error 2e-4 on logits of magnitude 4); ops.H2 = two fp16 planes of (value x power of two), 3 MMAs per product,
    # ~2^-22 relative, i.e. fp32-faithful — for the embedding / warp networks, whose output the sampler differentiates (an
    # error of 1e-4 in the embedding moves the image by 1e-2), and for the source-pass networks.  Three bf16 planes (6 MMAs,
    # the round-1 setting of those networks) give the same accuracy at twice the MMAs (tests/test_conv_modes_gpu.py) and
    # remain available through `precision=`.  The decoder's input planes are written by grid_sample_3d in bf16 (or, with
    # decoder=ops.H1, as one fp16 plane).
    PRECISION = dict(head_pose=ops.H2, expression=ops.H2, idt=ops.H2, warp=ops.H2, local_encoder=ops.H2, volume_source=ops.H2,
                     unet3d=ops.H2, decoder=2)
    # Named settings of `precision=`: "exact" is PRECISION; "fast" runs the decoder on one fp16 plane (ops.H1: one MMA per
    # product instead of three).  Fast mode keeps every uint8 output pixel within one level of the exact path
    # (tools/decoder_precision_emulation.py, tests/test_fast_decoder_gpu.py; INTEGRATION.md "Fast mode").
    PRESETS = dict(exact={}, fast=dict(decoder=ops.H1))
    # The source-volume networks on one fp16 plane (InferenceWrapper(source_precision="fast")).  Their output is the latent
    # volume's values, which the sampler and the decoder treat linearly or contract: the same error size as the decoder's fast
    # mode (tools/decoder_precision_emulation.py --source; DESIGN.md section 2).  The source volume is cached for a whole clip,
    # so its error is a fixed bias in every frame: this is a setting of its own, not part of PRESETS["fast"].
    SOURCE_FAST = dict(local_encoder=ops.H1, volume_source=ops.H1, unet3d=ops.H1)
    # networks whose output feeds the sampler's coordinates: never on one plane
    SAMPLER_NETS = ("head_pose", "expression", "idt", "warp")

    @classmethod
    def resolve_precision(cls, precision) -> dict:
        """`precision=` of Model: None, a preset name ("exact" / "fast") or a dict of per-network overrides of PRECISION"""
        if precision is None or isinstance(precision, str):
            if (precision or "exact") not in cls.PRESETS:
                raise ValueError(f"precision={precision!r}: the named settings are {sorted(cls.PRESETS)}")
            precision = cls.PRESETS[precision or "exact"]
        pr = dict(cls.PRECISION)
        pr.update(precision)
        if pr["decoder"] == ops.H2:
            raise ValueError("the decoder's input planes are written by grid_sample_3d in bf16 or as one fp16 plane; it runs "
                             "with 2 or 3 bf16 planes or ops.H1")
        one_plane = sorted(net for net in cls.SAMPLER_NETS if pr[net] == ops.H1)
        if one_plane:
            raise ValueError(f"ops.H1 (one fp16 plane) is not for {one_plane}: the head-pose, expression, identity and warp "
                             "networks feed the sampler's coordinates, which amplify their errors ~100x (DESIGN.md section 2)")
        return pr

    def __init__(self, cfg: HotPathConfig, state_dict, head_pose_state_dict, device="cuda", precision=None):
        """precision: None / "exact" (PRECISION), "fast" (decoder on ops.H1), or a dict overriding PRECISION per network
        (SOURCE_FAST puts the local encoder, the source volume blocks and the 3-D U-Net on ops.H1)."""
        self.cfg = cfg
        dev = torch.device(device)
        sd = state_dict
        pr = self.resolve_precision(precision)
        self.precision = pr
        self.local_encoder_nw = nets.LocalEncoder(sd, cfg, dev, planes=pr["local_encoder"])
        self.idt_embedder_nw = nets.IdtEmbed(sd, cfg, dev, planes=pr["idt"])
        self.expression_embedder_nw = nets.ExpressionEmbed(sd, cfg, dev, planes=pr["expression"])
        self.predict_embed = nets.PredictEmbed(sd, cfg, dev)
        self.xy_generator_nw = nets.WarpGenerator(sd, "xy_generator_nw", cfg, dev, planes=pr["warp"])
        self.uv_generator_nw = nets.WarpGenerator(sd, "uv_generator_nw", cfg, dev, planes=pr["warp"])
        self.volume_source_nw = nets.VolumeSource(sd, cfg, dev, planes=pr["volume_source"]) if cfg.source_volume_num_blocks > 0 else None
        self.volume_process_nw = nets.Unet3D(sd, cfg, dev, planes=pr["unet3d"])
        self.decoder_nw = nets.Decoder(sd, cfg, dev, planes=pr["decoder"])
        self.head_pose_regressor = nets.HeadPoseRegressor(head_pose_state_dict, dev, planes=pr["head_pose"])
        self.device = dev

    # ---- notebooks/infer.py:374-507 ----
    @torch.no_grad()
    def source_pass(self, src: torch.Tensor, taps: Optional[dict] = None, pose_override=None,
                    mask: Optional[torch.Tensor] = None, c_source_latent_volume: Optional[torch.Tensor] = None,
                    c_target_latent_volume: Optional[torch.Tensor] = None):
        """src (1,3,H,W) fp32 in [0,1] on device.  Returns the cached source state.
        mask (1,1,H,W) or None (= ones): the identity embedder and the local encoder see src * mask (infer.py:425-426);
        the head-pose regressor (:430) and the expression embedder (called with use_seg=False, :455) see src itself.
        c_source_latent_volume / c_target_latent_volume (1,C,D,S,S) replace the volumes where the reference substitutes
        them (:491, :500).
        pose_override = (theta (1,4,4), warp (1,3,4), align2d (1,2,3)) replaces the on-device pose algebra (tests only:
        lets a parity test inject the reference's own fp32 matrices, see tests/test_model_gpu.py)."""
        cfg = self.cfg
        src = src.contiguous().float()
        masked = src if mask is None else (src * mask.to(self.device).float()).contiguous()
        ops.begin_pass(self.device)
        st = SimpleNamespace()
        st.idt_embed = self.idt_embedder_nw(masked)                    # (1,512,4,4) NCHW
        vol = self.local_encoder_nw(masked)                            # (1,D,S,S,C)
        srt = self.head_pose_regressor(src)
        st.pred_source_theta, inv_warp, align = ops.pose_theta(srt, invert_warp=True)
        if pose_override is not None:
            st.pred_source_theta, inv_warp, align = [t.to(self.device).float().contiguous() for t in pose_override]
        st.source_theta_dev = st.pred_source_theta[0].contiguous()
        pose_embed, _ = self.expression_embedder_nw(src, align)
        st.pred_source_pose_embed = pose_embed
        E = self.predict_embed(pose_embed, st.idt_embed)
        xy_warp = self.xy_generator_nw(E)                              # (1,D,S,S,3)
        if self.volume_source_nw is not None:
            vol = self.volume_source_nw(vol)
        if c_source_latent_volume is not None:
            vol = self._volume_cl(c_source_latent_volume)
        st.source_latent_volume = vol
        st.source_rotation_warp_theta = inv_warp
        st.source_xy_warp_resize = xy_warp
        v = ops.grid_sample3d(vol, theta=inv_warp, out_size=(cfg.D, cfg.S, cfg.S), in_layout="cl")
        v = ops.grid_sample3d(v, grid=xy_warp, in_layout="cl")
        if c_target_latent_volume is not None:
            v = self._volume_cl(c_target_latent_volume)
        st.target_latent_volume_1 = v
        st.target_latent_volume = self.volume_process_nw(v)           # (1,D,S,S,C) channels-last
        if taps is not None:
            taps.update(srt_source=srt, source_pose_embed=pose_embed, source_embed=E, xy_warp=xy_warp)
        return st

    def _volume_cl(self, vol: torch.Tensor) -> torch.Tensor:
        """caller-supplied latent volume in the reference's (1,C,D,S,S) layout -> channels-last (1,D,S,S,C) on device"""
        cfg = self.cfg
        if tuple(vol.shape) != (1, cfg.C, cfg.D, cfg.S, cfg.S):
            raise ValueError(f"latent volume must be (1,{cfg.C},{cfg.D},{cfg.S},{cfg.S}), got {tuple(vol.shape)}")
        return vol.to(self.device).float().permute(0, 2, 3, 4, 1).contiguous()

    # ---- notebooks/infer.py:511-644 ----
    @torch.no_grad()
    def driver_pass(self, st, drv: torch.Tensor, mix: bool = True, target_theta: bool = True, taps: Optional[dict] = None,
                    want_logits: bool = False, pose_override=None, mix_old: bool = False,
                    custom_srt: Optional[torch.Tensor] = None, custom_pose_embed: Optional[torch.Tensor] = None,
                    smooth_state: Optional[torch.Tensor] = None, smooth_momentum: float = 0.5, smooth_init: bool = False,
                    encode_only: bool = False, pose_only: bool = False, pose_in: Optional[tuple] = None):
        """drv (1,3,H,W) fp32 on device -> (img (1,3,H,W), feat_2d, img_feat, state).
        mix / mix_old: get_mixing_theta (infer.py:569-570, 686-736).  custom_srt (1,9) = the caller's
        custome_target_theta_embed (scale, rotation, translation) replacing the regressed pose (:566-567).
        custom_pose_embed (1,128) replaces the expression embedding (:602-603).  smooth_state (3,4) on device: the
        wrapper's self.theta, smoothed in place with smooth_momentum (smooth_pose=True, :571-581).
        drv=None (both custom_srt and custom_pose_embed given): an image-free frame, without the head-pose regressor and the
        expression encoder; state.srt is then custom_srt.  encode_only: stop after the expression encoder and return
        (None, None, None, state): the frame's regressed pose state.srt and its embedding state.target_pose_embed, whose 2-D
        alignment comes from the mixed pose (so it depends on mix / mix_old and, with mix, on st's source pose).
        A smoothing frame in flight (DriverPipeline(smooth=True)) runs in two parts around its pose step, the one launch that
        carries state from frame to frame.  pose_only: stop after the pose algebra and return (None, None, None, state) with
        state.pred_target_theta the (1,4,4) pose, mixed and not smoothed, and state.srt.  pose_in = (theta (1,4,4), warp
        (1,3,4), align (1,2,3)): the pose step already wrote the frame's pose there; skip the head-pose regressor and the pose
        algebra and run the rest of the frame on it (state.srt is then None)."""
        cfg = self.cfg
        if drv is None and (custom_pose_embed is None or (custom_srt is None and pose_in is None) or encode_only
                            or taps is not None):
            raise ValueError("driver_pass: a frame without a driver image needs custom_srt and custom_pose_embed")
        if pose_in is not None and (pose_only or smooth_state is not None or pose_override is not None):
            raise ValueError("driver_pass: pose_in is the frame's finished pose; it takes no pose_only, smoothing or override")
        if drv is not None:
            drv = drv.contiguous().float()
        ops.begin_pass(self.device)
        if pose_in is not None:
            srt = None
            theta, warp, align = pose_in
        else:
            srt = None if drv is None else self.head_pose_regressor(drv)
            srt_used = srt if custom_srt is None else custom_srt.to(self.device).float().reshape(1, 9).contiguous()
            if srt is None:
                srt = srt_used     # an image-free frame reports the supplied pose
            theta, warp, align = ops.pose_theta(srt_used, source_theta=st.source_theta_dev if mix else None, mix=mix,
                                                mix_old=mix_old, smooth_state=smooth_state, smooth_momentum=smooth_momentum,
                                                smooth_init=smooth_init)
        if pose_override is not None:
            theta, warp, align = [t.to(self.device).float().contiguous() for t in pose_override]
        if pose_only:
            return None, None, None, SimpleNamespace(pred_target_theta=theta, target_pose_embed=None, srt=srt)
        if custom_pose_embed is not None and taps is None:
            pose_embed, aligned = None, None      # the expression encoder's output would be discarded (infer.py:602-603)
        else:
            pose_embed, aligned = self.expression_embedder_nw(drv, align, want_aligned=taps is not None)
        if encode_only:
            return None, None, None, SimpleNamespace(pred_target_theta=theta, target_pose_embed=pose_embed, srt=srt)
        if not target_theta:
            warp = st.pred_source_theta[:, :3].contiguous()
        if custom_pose_embed is not None:
            pose_embed = custom_pose_embed.to(self.device).float().reshape(1, -1).contiguous()
        E = self.predict_embed(pose_embed, st.idt_embed)
        uv_warp = self.uv_generator_nw(E)
        v = ops.grid_sample3d(st.target_latent_volume, grid=uv_warp, in_layout="cl")
        feat = ops.grid_sample3d(v, theta=warp, out_size=(cfg.D, cfg.S, cfg.S), in_layout="cl", out_layout="hwdc",
                                 want_f32=taps is not None, want_split=True, planes=self.decoder_nw.planes)
        if taps is not None:
            aligned_vol, feat = feat
            taps.update(srt=srt, theta=warp, pose_embed=pose_embed, embed=E, uv_warp=uv_warp, aligned_face=aligned,
                        aligned_volume_hwdc=aligned_vol)
        feat2d = feat.view(1, 1, cfg.S, cfg.S, cfg.D * cfg.C)
        img, deep_f, img_f = self.decoder_nw(feat2d, want_logits=want_logits)
        st_out = SimpleNamespace(pred_target_theta=theta, target_pose_embed=pose_embed, srt=srt)
        return img, deep_f, img_f, st_out


    @staticmethod
    def check_inputs(image: bool, theta_embed: bool, pose_embed: bool, encode: bool) -> None:
        """ValueError unless the inputs a captured frame reads are a valid set: a driver image, and / or the caller's
        pose (theta_embed) and expression embedding (pose_embed); an image-free frame takes both, an encoding frame
        (encode: the pose and the embedding of its image, no rendering) only the image"""
        if not image and not (theta_embed and pose_embed):
            raise ValueError("a frame without a driver image needs both theta_embed and pose_embed")
        if encode and not (image and not theta_embed and not pose_embed):
            raise ValueError("an encoding frame reads a driver image and nothing else")

    def check_refine(self, refine, encode: bool) -> None:
        """ValueError unless `refine` (a stage2.Stage2Model or None) can follow this model's frames in one graph"""
        if refine is None:
            return
        if encode:
            raise ValueError("an encoding frame renders no image to refine: refine needs encode=False")
        if ops._dev_key(refine.device) != ops._dev_key(self.device):
            raise ValueError(f"the stage-2 model is on {refine.device}, the stage-1 model on {self.device}: refined frames run "
                             "both on one device")

    @staticmethod
    def check_refine_masks(refine, refine_masks: Optional[dict] = None, composite=None) -> None:
        """ValueError unless stage 2's mask networks refine_masks (dict(modnet=, face_idt=, cloth=), Stage2Model.refine) and the
        compositing matte network `composite` can run in a refined frame of `refine`"""
        if refine is None:
            if refine_masks or composite is not None:
                raise ValueError("refine_masks= and composite= act on stage 2: they need refine=")
            return
        if composite is not None and not callable(composite):
            raise ValueError(f"composite must be a callable img (1,3,H,W) -> matte (1,1,H,W), got {type(composite).__name__}")
        rm = dict(refine_masks or {})
        if set(rm) - {"modnet", "face_idt", "cloth"}:
            raise ValueError(f"refine_masks takes modnet, face_idt and cloth, got {sorted(rm)}")
        if rm.get("modnet") is not None and not callable(rm["modnet"]):
            raise ValueError(f"refine_masks['modnet'] must be the matting network (a callable), got {type(rm['modnet']).__name__}")
        if rm.get("face_idt") is not None:
            if rm.get("modnet") is None:
                raise ValueError("stage 2's face mask multiplies the MODNet matte: refine_masks needs modnet with face_idt")
            if not callable(getattr(rm["face_idt"], "label_masks", None)):
                raise ValueError("refine_masks['face_idt'] must be a masks.FaceParsing: a captured frame keeps its uint8 label masks")

    def make_driver_graph(self, st, mix: bool = True, target_theta: bool = True, slot: int = 0, mix_old: bool = False,
                          smooth_state: Optional[torch.Tensor] = None, smooth_momentum: float = 0.5, image: bool = True,
                          theta_embed: bool = False, pose_embed: bool = False, encode: bool = False, refine=None,
                          refine_masks: Optional[dict] = None, composite=None, pose_step: bool = False):
        """Capture one driver frame (all ~240 kernel launches) into a CUDA graph: removes the Python/ctypes launch
        overhead from the per-frame loop.  Returns replay(drv (1,3,H,W) on device) -> img (1,3,H,W) (static buffer).
        The graph reads its identity from buffers of its own (replay.identity, dist.new_identity), never from `st`:
        `st` is loaded into them before the capture, and replay.load(other) switches the identity of later replays without
        a new capture.
        `slot` selects the scratch set (ops.set_slot) the captured frame uses; graphs that may replay concurrently on
        different streams need different slots.  smooth_state (3,4): the captured frame also smooths its pose into this
        tensor in place (smooth_pose=True, infer.py:571-581; the state must already be seeded by one eager frame) - frames of
        such a graph are a recurrence and must replay one after the other on one stream.
        The inputs the graph reads (check_inputs), each from a static buffer of its own that the caller fills before a
        replay: image -> replay.static_in (1,3,H,W); theta_embed -> replay.static_theta (1,9), the caller's (scale,
        rotation, translation) in place of the regressed pose; pose_embed -> replay.static_pose (1,E), the caller's
        expression embedding (the expression encoder is then not captured).  Without an image the head-pose regressor is
        not captured either.  encode: the graph stops after the expression encoder (driver_pass(encode_only=True)):
        replay.static_state.srt / .target_pose_embed are the frame's pose and embedding, static_out is None, and its
        identity buffers hold only the source pose, the one identity field the embedding depends on.
        refine (a stage2.Stage2Model on this device): the graph continues with stage 2 on the frame's image
        (Stage2Model.refine, the stage-2 wrapper's default masks): replay.static_out is then the refined (1,3,S2,S2) image,
        replay.static_u8 its (1,S2,S2,3) uint8 frame and replay.static_stage1 the stage-1 image.  The warm-up passes run
        stage 2 under the same scratch set, so its workspaces exist before the capture.
        refine_masks (dict(modnet=, face_idt=, cloth=), with refine): stage 2 runs with the masks these networks give
        (Stage2Model.refine), the stage-2 wrapper's masks when they are plugged into it.  composite (a callable img (1,3,H,W) ->
        matte (1,1,H,W), with refine, e.g. masks.face_matte): the stage-1 image is composited over replay.static_bg (3,H,W),
        which the caller fills before a replay, as video.connect_img_and_bg does, before stage 2.  The caller's networks are
        captured with the frame (INTEGRATION.md "Mask networks in captured frames": no host syncs, static shapes, already on
        this device); the warm-up passes run them too.  A capture that fails raises RuntimeError naming the network that
        broke it.
        pose_step: the frame is captured as two graphs around its pose step, for frames whose poses are smoothed in flight
        (DriverPipeline(smooth=True)).  replay.head_graph runs the input side up to the pose algebra, mixed but not smoothed,
        into replay.static_mixed (1,4,4); the caller then runs Model.pose_step from it into replay.pose (theta (1,4,4), warp
        (1,3,4), align (1,2,3)), and replay.graph runs the rest of the frame from there.  Not with smooth_state or encode."""
        self.check_inputs(image, theta_embed, pose_embed, encode)
        self.check_refine(refine, encode)
        self.check_refine_masks(refine, refine_masks, composite)
        self.check_pose_step(pose_step, encode, smooth_state)
        prev = ops.set_slot(slot)
        try:
            return self._make_driver_graph(st, mix, target_theta, mix_old, smooth_state, smooth_momentum, image, theta_embed,
                                           pose_embed, encode, refine, refine_masks, composite, pose_step)
        finally:
            ops.set_slot(prev)

    @staticmethod
    def check_pose_step(pose_step: bool, encode: bool, smooth_state=None) -> None:
        """ValueError unless a frame split at its pose step (make_driver_graph(pose_step=True)) can take these options"""
        if pose_step and encode:
            raise ValueError("smoothing frames in flight render their frames: smooth needs encode=False")
        if pose_step and smooth_state is not None:
            raise ValueError("a frame split at its pose step is smoothed by the pose step, not in the graph: no smooth_state")

    @staticmethod
    def pose_step(mixed: torch.Tensor, state: torch.Tensor, momentum: float, init: bool, out: tuple):
        """The pose step of a smoothing frame in flight, between its two graphs: smooths the frame's mixed pose (1,4,4) into
        the (3,4) state in place (seeding it first if init, the reference's `self.theta is None`), and writes the smoothed
        pose, its warp and 2-D alignment into `out`.  driver_pass's pose algebra keeps the mixed pose in fp32 and rereads
        it here unchanged, so this launch smooths, inverts and aligns exactly what one smoothing launch would."""
        return ops.pose_theta(None, theta_in=mixed, smooth_state=state, smooth_momentum=momentum, smooth_init=init, out=out)

    def _make_driver_graph(self, st, mix, target_theta, mix_old=False, smooth_state=None, smooth_momentum=0.5, image=True,
                           theta_embed=False, pose_embed=False, encode=False, refine=None, refine_masks=None, composite=None,
                           pose_step=False):
        s, dev = self.cfg.image_size, self.device
        static_in = torch.zeros((1, 3, s, s), dtype=torch.float32, device=dev) if image else None
        # the warm-up passes run on the unit pose (scale 1, no rotation or translation) and a zero embedding
        static_theta = torch.tensor([[1.0, 1, 1, 0, 0, 0, 0, 0, 0]], device=dev) if theta_embed else None
        static_pose = torch.zeros((1, self.cfg.expr_channels), dtype=torch.float32, device=dev) if pose_embed else None
        fields = ("pred_source_theta",) if encode else tuple(source_state_shapes(self.cfg))
        identity = new_identity(self.cfg, dev, fields)
        kw = dict(mix=mix, target_theta=target_theta, mix_old=mix_old, custom_srt=static_theta, custom_pose_embed=static_pose,
                  encode_only=encode)
        if smooth_state is not None:
            kw.update(smooth_state=smooth_state, smooth_momentum=smooth_momentum, smooth_init=False)
            saved = smooth_state.clone()  # the warm-up and capture passes smooth a dummy frame into the state: put it back after
        # a frame split at its pose step: the pose buffers the step writes and the tail reads, and a state for the warm-up
        pose = tuple(torch.zeros(shp, dtype=torch.float32, device=dev) for shp in ((1, 4, 4), (1, 3, 4), (1, 2, 3))) \
            if pose_step else None
        warm_state = torch.zeros((3, 4), dtype=torch.float32, device=dev) if pose_step else None
        head_graph = head = None

        def replay(drv: torch.Tensor) -> torch.Tensor:
            if head_graph is not None:
                raise RuntimeError("a frame split at its pose step runs through DriverPipeline(smooth=True).submit(..., track=)")
            static_in.copy_(drv, non_blocking=True)
            graph.replay()
            return static_out

        # load must not refer to replay: a reference cycle would leave the graph to the cyclic garbage collector, which may
        # then destroy it in the middle of another graph's capture (and so invalidate that capture)
        loaded = [None]

        def load(state) -> None:
            """Make `state` the identity of the following replays: copy its identity fields into the graph's buffers on the
            current stream (nothing to do if it is loaded already).  The graph keeps a reference to the loaded state, and
            its tensors are marked as in use by the current stream, so a caller may drop the state before the copy ran."""
            if loaded[0] is state:
                return
            check_identity(state, self.cfg)
            cur = torch.cuda.current_stream(self.device)
            for k in fields:
                src = getattr(state, k)
                getattr(identity, k).copy_(src, non_blocking=True)
                if src.is_cuda:
                    src.record_stream(cur)
            loaded[0] = state

        replay.load, replay.identity = load, identity
        load(st)  # the warm-up and capture passes run on a real identity
        static_bg = torch.zeros((3, s, s), dtype=torch.float32, device=dev) if composite is not None else None
        culprit = []   # the caller's network that raised, if one did
        refine_kw = _named_networks(dict(refine_masks or {}), composite, culprit)

        def refined(img):
            if refine_kw.get("composite") is not None:
                matte = refine_kw["composite"](img)
                if not isinstance(matte, torch.Tensor) or tuple(matte.shape) != (1, 1, s, s):
                    got = tuple(matte.shape) if isinstance(matte, torch.Tensor) else type(matte).__name__
                    raise ValueError(f"composite must return the matte (1,1,{s},{s}), got {got}")
                return refine.refine(img, matte=matte, bg=static_bg, **{k: v for k, v in refine_kw.items() if k != "composite"})
            return refine.refine(img, **refine_kw)

        def warm_frame():
            if not pose_step:
                return self.driver_pass(identity, static_in, **kw)[0]
            mixed = self.driver_pass(identity, static_in, pose_only=True, **kw)[3].pred_target_theta
            self.pose_step(mixed, warm_state, 0.5, True, pose)
            return self.driver_pass(identity, static_in, pose_in=pose, **kw)[0]

        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        try:
            with torch.cuda.stream(side):
                for _ in range(2):
                    img = warm_frame()
                    if refine is not None:
                        refined(img)
            torch.cuda.current_stream(self.device).wait_stream(side)
            torch.cuda.synchronize(self.device)
            if pose_step:
                head_graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(head_graph):
                    head = self.driver_pass(identity, static_in, pose_only=True, **kw)[3]
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self.driver_pass(identity, static_in, pose_in=pose, **kw)
                static_out = static_stage1 = out[0]
                static_u8 = None
                if refine is not None:
                    _, static_out, static_u8 = refined(static_stage1)
        except Exception as e:
            if not culprit:
                raise
            raise RuntimeError(f"the refined driver frame could not be captured: {culprit[0]} raised {type(e).__name__}: {e}.  "
                               "A network in a captured frame must issue no host syncs, keep its shapes static and already be "
                               "on this device (INTEGRATION.md \"Mask networks in captured frames\"); otherwise run stage 2 with "
                               "its masks eagerly, with stage2.InferenceWrapper.forward") from e
        if smooth_state is not None:
            smooth_state.copy_(saved)

        so = out[3]
        if pose_step:    # the frame's regressed (or supplied) pose comes from its head
            so = SimpleNamespace(pred_target_theta=so.pred_target_theta, target_pose_embed=so.target_pose_embed, srt=head.srt)
        replay.graph, replay.head_graph = graph, head_graph
        replay.static_mixed, replay.pose = (head.pred_target_theta if pose_step else None), pose
        replay.static_in, replay.static_out, replay.static_state = static_in, static_out, so
        replay.static_theta, replay.static_pose = static_theta, static_pose
        replay.static_stage1, replay.static_u8, replay.static_bg = static_stage1, static_u8, static_bg
        return replay


def _named_networks(refine_masks: dict, composite, culprit: list) -> dict:
    """Stage2Model.refine's mask arguments, plus `composite`, with every caller network wrapped so that an exception it raises
    first appends the network's name to `culprit` (make_driver_graph's capture error names it)"""
    def named(fn, name):
        def call(*a, **k):
            try:
                return fn(*a, **k)
            except Exception:
                culprit.append(name)
                raise
        return call

    out = dict(refine_masks)
    if out.get("modnet") is not None:
        out["modnet"] = named(out["modnet"], "the stage-2 matting network (modnet)")
    if out.get("face_idt") is not None:
        out["face_idt"] = copy.copy(out["face_idt"])
        out["face_idt"].net = named(out["face_idt"].net, "the stage-2 face parser (face_idt.net)")
    if composite is not None:
        out["composite"] = named(composite, "the compositing matte network (composite / mask_fn)")
    return out


class PoseTrack:
    """The pose-smoothing state of one stream of driver frames (one webcam, one participant of a call): the (3,4) fp32 state
    on the device (the reference wrapper's self.theta), the momentum it is smoothed with (theta * m + state * (1 - m),
    notebooks/infer.py:571-581), whether it is seeded, and the event of its last pose step.  Made by DriverPipeline.track;
    the first frame after creation or reset() seeds the state with its own pose.  momentum may be changed between frames:
    it is an argument of each pose step, not part of a captured graph."""

    def __init__(self, device, momentum: float = 0.5, state: Optional[torch.Tensor] = None):
        self.momentum = self.check_momentum(momentum)
        self.state = torch.zeros((3, 4), dtype=torch.float32, device=device) if state is None else state
        self.seeded = False
        self.event = None   # recorded after the track's last pose step; the next one waits for it

    @staticmethod
    def check_momentum(momentum) -> float:
        m = float(momentum)
        if not 0.0 <= m <= 1.0:
            raise ValueError(f"pose momentum must be in [0, 1], got {momentum!r}")
        return m

    def reset(self) -> None:
        """the next frame seeds the state (reset_tracking)"""
        self.seeded = False


class DriverPipeline:
    """Keeps `depth` driver frames in flight on one GPU.  Driver frames are independent given the cached source state
    (notebooks/infer.py:511-644 reads only self.* source tensors), and roughly a quarter of a frame is a chain of ~120
    tiny launches (head-pose and expression encoders at 4^2..56^2) that leaves most SMs idle; replaying the captured
    frames of consecutive inputs on alternating streams lets one frame's big decoder kernels fill those holes.
    Frame i's result is produced in order on stream i % depth; nothing is batched and every frame runs the same
    kernels as the single-stream path.

    Each slot's graph reads the identity from buffers of its own (Model.make_driver_graph), so frames of different
    identities may be in flight at once: submit(..., st=) names the source state a frame animates.  A slot whose loaded
    identity differs copies the new one in (~25 MB at 512^2) on its stream before the frame; nothing is re-captured.
    The slots use scratch sets of their own (scratch_slots), apart from the eager passes' set 0, so a source pass may run
    on the current stream while frames are in flight.

    image / theta_embed / pose_embed name the inputs every frame takes (Model.make_driver_graph): the driver image, and the
    caller's pose (1,9) and expression embedding (1,E) for the frame.  encode: each frame stops after the expression
    encoder; its pose and embedding are slot.run.static_state.srt / .target_pose_embed.

    refine (a stage2.Stage2Model): every frame is refined by stage 2 in the same graph (Model.make_driver_graph):
    slot.run.static_out is the refined (1,3,S2,S2) image, slot.run.static_u8 its uint8 frame and slot.run.static_stage1 the
    stage-1 image.  submit(..., u8_out=) copies the uint8 frame out on the frame's stream.
    refine_masks / composite: stage 2's mask networks and the compositing matte network (Model.make_driver_graph), captured
    with every frame; a compositing pipeline's frames take submit(..., bg=).

    smooth: every frame's pose is smoothed over the frames of its track (smooth_pose, notebooks/infer.py:571-581), with the
    frames still in flight.  Only one launch of a frame carries state from frame to frame, so each slot captures its frame
    as two graphs around it (Model.make_driver_graph(pose_step=True)); between them the frame's pose step
    (Model.pose_step) runs on the pipeline's pose stream, after the frame's head and after its track's previous pose step.
    submit order is the order of each track's recurrence.  Every frame names its track: submit(..., track=pipe.track()),
    one PoseTrack per incoming stream of frames."""

    def __init__(self, model: "Model", st, depth: int = 2, mix: bool = True, target_theta: bool = True, mix_old: bool = False,
                 image: bool = True, theta_embed: bool = False, pose_embed: bool = False, encode: bool = False, refine=None,
                 refine_masks: Optional[dict] = None, composite=None, smooth: bool = False):
        model.check_inputs(image, theta_embed, pose_embed, encode)
        model.check_refine(refine, encode)
        Model.check_refine_masks(refine, refine_masks, composite)
        Model.check_pose_step(smooth, encode)
        self.model, self.depth, self.n = model, depth, 0
        self.image, self.theta_embed, self.pose_embed, self.encode = image, theta_embed, pose_embed, encode
        self.refine, self.composite, self.smooth = refine, composite, smooth
        self.st = st  # the current identity: frames submitted without st= animate it
        # the pose steps of all the pipeline's frames, in submit order: only tiny launches run here
        self.pose_stream = torch.cuda.Stream(device=model.device) if smooth else None
        self.slots = []
        for k in self.scratch_slots(depth):
            run = model.make_driver_graph(st, mix=mix, target_theta=target_theta, slot=k, mix_old=mix_old, image=image,
                                          theta_embed=theta_embed, pose_embed=pose_embed, encode=encode, refine=refine,
                                          refine_masks=refine_masks, composite=composite, pose_step=smooth)
            self.slots.append(SimpleNamespace(run=run, stream=torch.cuda.Stream(device=model.device),
                                              done=torch.cuda.Event(), busy=False, bg=None))

    def track(self, momentum: float = 0.5) -> PoseTrack:
        """a new pose track on this pipeline's device (a smoothing pipeline's frames name theirs in submit(..., track=)); it
        may be used by several pipelines of the device, its frames then ordered by submit across them"""
        return PoseTrack(self.model.device, momentum)

    @staticmethod
    def scratch_slots(depth: int) -> list:
        """the scratch set (ops.set_slot) of each pipeline slot: 1 .. depth.  Set 0 belongs to the eager passes
        (Model.source_pass / driver_pass on the current stream), which may overlap frames in flight."""
        return [k + 1 for k in range(depth)]

    def _check_submit(self, drv, theta_embed, pose_embed, outs, u8_out=None, bg=None, track=None) -> None:
        """ValueError unless a frame's inputs are the ones the pipeline was captured for, of the right shapes, u8_out
        a (1,S2,S2,3) uint8 buffer of a refining pipeline, bg a (3,H,W) fp32 background of a compositing one and track a
        PoseTrack on this device, given exactly when the pipeline smooths"""
        if (track is not None) != bool(getattr(self, "smooth", False)):
            raise ValueError("track= names the pose track of a frame of a smoothing pipeline (smooth=True): give it exactly when "
                             "the pipeline smooths")
        if track is not None:
            if not isinstance(track, PoseTrack):
                raise ValueError(f"track must be a PoseTrack (DriverPipeline.track()), got {type(track).__name__}")
            if ops._dev_key(track.state.device) != ops._dev_key(self.model.device):
                raise ValueError(f"the track's state is on {track.state.device}, the pipeline on {self.model.device}")
            PoseTrack.check_momentum(track.momentum)
        if (bg is not None) != (getattr(self, "composite", None) is not None):
            raise ValueError("bg= is the background of a compositing pipeline (composite=): give it exactly when the pipeline "
                             "composites")
        if bg is not None:
            s = self.model.cfg.image_size
            if not isinstance(bg, torch.Tensor) or tuple(bg.shape) != (3, s, s) or bg.dtype != torch.float32:
                got = (tuple(bg.shape), bg.dtype) if isinstance(bg, torch.Tensor) else type(bg).__name__
                raise ValueError(f"bg must be a float32 tensor of shape {(3, s, s)}, got {got}")
        if u8_out is not None:
            if self.refine is None:
                raise ValueError("u8_out: only a refining pipeline (refine=) writes a uint8 frame")
            s2 = self.refine.cfg.output_size
            if not isinstance(u8_out, torch.Tensor) or tuple(u8_out.shape) != (1, s2, s2, 3) or u8_out.dtype != torch.uint8 \
                    or not u8_out.is_contiguous():
                got = (tuple(u8_out.shape), u8_out.dtype) if isinstance(u8_out, torch.Tensor) else type(u8_out).__name__
                raise ValueError(f"u8_out must be a contiguous uint8 tensor of shape {(1, s2, s2, 3)}, got {got}")
        given = dict(image=drv is not None, theta_embed=theta_embed is not None, pose_embed=pose_embed is not None)
        want = dict(image=self.image, theta_embed=self.theta_embed, pose_embed=self.pose_embed)
        if given != want:
            raise ValueError(f"this pipeline was captured for the inputs {sorted(k for k, v in want.items() if v)}, "
                             f"got {sorted(k for k, v in given.items() if v)}")
        shapes = dict(theta_embed=(theta_embed, (1, 9)), pose_embed=(pose_embed, (1, self.model.cfg.expr_channels)))
        for name, (t, shp) in shapes.items():
            if t is not None and (not isinstance(t, torch.Tensor) or tuple(t.shape) != shp):
                got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
                raise ValueError(f"{name} must be a tensor of shape {shp}, got {got}")
        if self.encode and any(o is not None for o in outs):
            raise ValueError("an encoding pipeline renders no image: host_out / dev_out must be None")

    def submit(self, drv: Optional[torch.Tensor], host_out: Optional[torch.Tensor] = None, dev_out: Optional[torch.Tensor] = None,
               st=None, theta_embed: Optional[torch.Tensor] = None, pose_embed: Optional[torch.Tensor] = None,
               u8_out: Optional[torch.Tensor] = None, bg: Optional[torch.Tensor] = None, track: Optional[PoseTrack] = None):
        """Queue one frame (device tensor, or pinned host tensor -> asynchronous H2D on the frame's stream).  If `host_out`
        (pinned) / `dev_out` is given the image is copied into it on the same stream.  Returns a ticket: ticket.done is an
        event recorded when this frame (and its copy-out) has finished (ticket.slot.done is the same event, i.e. always the
        slot's latest frame); slot.run.static_out is valid until the slot's next submit.  A slot's frames are ordered by
        its stream, so a caller may queue further frames on a busy slot — it only has to keep the host_out / dev_out
        buffers of unfinished frames apart.
        st: the source state (Model.source_pass, dist.broadcast_source_state) to animate; it becomes the pipeline's
        current identity.  None: the current identity.  The frame's stream waits for the current stream first, so a
        state whose source pass was just queued there may be given at once, and the caller may drop it after this call.
        theta_embed (1,9) / pose_embed (1,E): the frame's pose and expression embedding, for a pipeline captured to take
        them; they are copied into the slot's buffers on its stream like the image.  drv is None for an image-free
        pipeline.  Inputs other than the pipeline's, or of other shapes, raise ValueError before anything is queued.
        u8_out (1,S2,S2,3) uint8, pinned host or device (a refining pipeline only): the refined frame's uint8 image
        (slot.run.static_u8) is copied into it on the frame's stream, before ticket.done.
        bg (3,H,W) fp32 (a compositing pipeline only, and then for every frame): the background the frame is composited over.  A
        slot copies it into its buffer (slot.run.static_bg) on its stream only when it is a different tensor from the slot's
        last one; the slot keeps a reference to it and marks it as in use by its stream, as replay.load does an identity.
        track (a smoothing pipeline only, and then for every frame): the PoseTrack whose state the frame's pose is smoothed
        into.  The frame's pose step waits for its head and for the track's last pose step, on any pipeline; the state is
        seeded by the track's first frame after creation or reset(), and smoothed with track.momentum as it is at submit."""
        if st is not None:
            check_identity(st, self.model.cfg)
        self._check_submit(drv, theta_embed, pose_embed, (host_out, dev_out), u8_out, bg, track)
        if st is not None:
            self.st = st
        sl = self.slots[self.n % self.depth]
        self.n += 1
        # a strided host tensor would otherwise take torch's staged, synchronous copy path
        inputs = [(buf, t if t.is_contiguous() else t.contiguous()) for buf, t in
                  ((sl.run.static_in, drv), (sl.run.static_theta, theta_embed), (sl.run.static_pose, pose_embed)) if t is not None]
        sl.stream.wait_stream(torch.cuda.current_stream(self.model.device))
        with torch.cuda.stream(sl.stream), torch.no_grad():
            sl.run.load(self.st)
            if bg is not None and bg is not sl.bg:
                sl.run.static_bg.copy_(bg, non_blocking=True)
                if bg.is_cuda:
                    bg.record_stream(sl.stream)
                sl.bg = bg
            for buf, t in inputs:
                buf.copy_(t, non_blocking=True)
            if track is not None:
                self._pose_step(sl, track)
            sl.run.graph.replay()
            if host_out is not None:
                host_out.copy_(sl.run.static_out, non_blocking=True)
            if dev_out is not None:
                dev_out.copy_(sl.run.static_out, non_blocking=True)
            if u8_out is not None:
                u8_out.copy_(sl.run.static_u8, non_blocking=True)
            sl.done = torch.cuda.Event()
            sl.done.record()
        sl.busy = True
        return SimpleNamespace(done=sl.done, slot=sl, index=self.n - 1)

    def _pose_step(self, sl, track: PoseTrack) -> None:
        """on the slot's stream: the frame's head, then (on the pose stream) its pose step, which the tail waits for"""
        sl.run.head_graph.replay()
        head = torch.cuda.Event()
        head.record()
        with torch.cuda.stream(self.pose_stream):
            self.pose_stream.wait_event(head)
            if track.event is not None:
                self.pose_stream.wait_event(track.event)
            if track.state.is_cuda:
                track.state.record_stream(self.pose_stream)   # a caller may drop the track before its last step ran
            Model.pose_step(sl.run.static_mixed, track.state, track.momentum, not track.seeded, sl.run.pose)
            track.event = torch.cuda.Event()
            track.event.record()
        track.seeded = True
        sl.stream.wait_event(track.event)

    def drain(self):
        cur = torch.cuda.current_stream(self.model.device)
        for sl in self.slots:
            cur.wait_stream(sl.stream)
            sl.busy = False


class InferenceWrapper(torch.nn.Module):
    def __init__(self, experiment_name, which_epoch='latest', model_file_name='', use_gpu=True, num_gpus=1,
                 fixed_bounding_box=False, project_dir='./', folder='mp_logs', model_='va',
                 torch_home='', debug=False, print_model=False, print_params=True, args_overwrite={}, state_dict=None,
                 pose_momentum=0.5, rank=0, args_path=None, head_pose_state_dict=None, precision="exact",
                 source_precision="exact"):
        """precision: "exact" (default: the parity path) or "fast" (the decoder on one fp16 plane: every uint8 output pixel
        within one level of "exact", INTEGRATION.md "Fast mode").  Every driver path (captured pipelines, the list form of
        forward, video.drive_image_with_video) runs with the model's setting.
        source_precision: "exact" (default) or "fast" (the source pass's local encoder, volume blocks and 3-D U-Net on one
        fp16 plane, Model.SOURCE_FAST; every uint8 pixel within one level of "exact").  Independent of `precision=`: the
        source volume is cached, so its error is the same in every frame of a clip."""
        super().__init__()
        if precision not in ("exact", "fast"):
            raise ValueError(f"precision={precision!r}: 'exact' or 'fast'")
        if source_precision not in ("exact", "fast"):
            raise ValueError(f"source_precision={source_precision!r}: 'exact' or 'fast'")
        if not use_gpu or not torch.cuda.is_available():
            raise RuntimeError("emoportraits_b200.InferenceWrapper needs a CUDA device (H100); there is no CPU path")
        if model_ != 'va':
            raise NotImplementedError(f"model_={model_!r}: only the stage-1 'va' model is implemented")
        self.use_gpu, self.debug, self.num_gpus, self.rank = use_gpu, debug, num_gpus, rank
        args_path = pathlib.Path(project_dir) / folder / experiment_name / 'args.txt' if args_path is None else args_path
        self.args = parse_args(args_path)
        self.args.project_dir = project_dir
        for k, v in (args_overwrite or {}).items():
            setattr(self.args, k, v)
        self.cfg = hot_path_config(self.args)
        self.device = torch.device('cuda', torch.cuda.current_device())

        self.model_checkpoint = pathlib.Path(project_dir) / folder / experiment_name / 'checkpoints' / model_file_name
        if state_dict is None:
            state_dict = torch.load(self.model_checkpoint, map_location='cpu')
        self.model_dict = state_dict
        if head_pose_state_dict is None:
            hp = getattr(self.args, 'head_pose_regressor_path', None)
            if not hp or not pathlib.Path(str(hp)).exists():
                raise FileNotFoundError(f"head pose regressor checkpoint not found ({hp}); pass head_pose_state_dict=")
            head_pose_state_dict = torch.load(hp, map_location='cpu')
        self.precision, self.source_precision = precision, source_precision
        model_precision = precision
        if source_precision == "fast":
            model_precision = dict(Model.PRESETS[precision], **Model.SOURCE_FAST)
        self.model = Model(self.cfg, state_dict, head_pose_state_dict, self.device, precision=model_precision)
        if rank == 0 and print_params:
            n = sum(v.numel() for v in state_dict.values())
            print(f'Number of parameters/buffers in checkpoint: {n}')

        # face tracking / smoothing state kept for API parity (notebooks/infer.py:159-177)
        self.fixed_bounding_box = fixed_bounding_box
        self.momentum = 0.01
        self.center = None
        self.size = None
        self.pose_momentum = pose_momentum
        self.theta = None
        self.norm_momentum = 0.1
        self.delta_yaw = None
        self.delta_pitch = None
        self.resize_warp = False
        self.use_seg = getattr(self.args, 'use_seg', True)
        self._state = None
        self._pipelines = OrderedDict()   # captured DriverPipelines by options, least recently used first
        self._smooth_graph = None
        self._track = None                # the PoseTrack of smoothed frames in flight: its state is self.theta
        # external mask networks (separate checkouts in the reference: repos/face_par_off behind model.face_idt, infer.py:410;
        # repos/MODNet, infer.py:140-149): None until the caller plugs them in (masks.FaceParsing(None, net=...), any MODNet module)
        self.face_idt = None
        self.modnet = None

    def get_mask(self, img):
        """notebooks/infer.py:649-684: MODNet matte of img (N,3,h,w) in [0,1]; normalisation and both 'area' resizes on the device."""
        from .masks import modnet_get_mask

        if self.modnet is None:
            raise NotImplementedError("get_mask needs the external MODNet network: set wrapper.modnet = <module>")
        return modnet_get_mask(self.modnet, img.to(self.device))

    @property
    def identity(self):
        """The current identity, as an opaque handle: the source state of the last source pass, or the handle assigned last.
        Assigning a handle read earlier makes its identity current again with no source pass and no graph capture: the
        cached source attributes (idt_embed, pred_source_theta, target_latent_volume, source_image, ...) return to it and
        the next driver frames animate it.  Each handle kept keeps its identity resident on the device: about 3 x 25 MB at
        512^2 (the source, warped and processed latent volumes)."""
        return self._state

    @identity.setter
    def identity(self, st):
        check_identity(st, self.cfg)
        if not hasattr(st, "wrapper_inputs"):
            raise ValueError("identity: assign a handle read from InferenceWrapper.identity (it carries the source image and "
                             "mask of its source pass)")
        self._use_identity(st)

    def _use_identity(self, st):
        self._state = st
        for k, v in st.wrapper_inputs.items():   # source_image, source_img_mask, ... as the source pass's forward set them
            setattr(self, k, v)
        # cached attributes of the reference wrapper (infer.py:405-507)
        self.idt_embed = st.idt_embed
        self.pred_source_theta = st.pred_source_theta
        self.pred_source_pose_embed = st.pred_source_pose_embed
        self.source_latent_volume = st.source_latent_volume.permute(0, 4, 1, 2, 3)       # NCDHW views
        self.source_xy_warp_resize = st.source_xy_warp_resize
        self.target_latent_volume_1 = st.target_latent_volume_1.permute(0, 4, 1, 2, 3)
        self.target_latent_volume = st.target_latent_volume.permute(0, 4, 1, 2, 3)

    # Captured pipelines a wrapper keeps, one per set of options (pose options, the inputs a frame takes, encoding or
    # rendering); the least recently used is dropped for a new one.  Plain frames, encode(), animate() and forward with an
    # embedding then alternate with no capture.
    PIPELINES = 4
    # Frames in flight of a refining pipeline (forward_refined).  Stage 2 at batch 1 @1024^2 fills an H100 on its own:
    # two, three and four frames in flight run within 1 % of each other (tools/refine_stream_bench.py, DESIGN.md section 7),
    # while every slot holds ~4 GB (exact) of captured activations.  Two keep one frame's host-side work under the other's.
    REFINE_DEPTH = 2

    def _driver_pipeline(self, mix, target_theta, mix_old, refine=None, refine_masks=None, composite=None, **inputs):
        """the captured four-in-flight pipeline of these options (DriverPipeline's image / theta_embed / pose_embed / encode,
        the stage-2 model that refines its frames, keyed with its precision, and the network objects of stage 2's masks and of
        the composite, with cloth); it serves every identity (submit(..., st=))"""
        key = (bool(mix), bool(target_theta), bool(mix_old), tuple(sorted(inputs.items())))
        if refine is not None:
            key += (("refine", refine, refine.precision),)
        if refine_masks or composite is not None:
            rm = refine_masks or {}
            key += (("masks", rm.get("modnet"), rm.get("face_idt"), bool(rm.get("cloth")), composite),)
        pipe = self._pipelines.pop(key, None)
        if pipe is None:
            depth = 4 if refine is None else self.REFINE_DEPTH
            pipe = DriverPipeline(self.model, self._state, depth=depth, mix=mix, target_theta=target_theta, mix_old=mix_old,
                                  refine=refine, refine_masks=refine_masks, composite=composite, **inputs)
        self._pipelines[key] = pipe
        # the new pipeline's captures synchronized the device, so nothing of a dropped one is still running
        while len(self._pipelines) > self.PIPELINES:
            self._pipelines.popitem(last=False)
        return pipe

    def _forward_list(self, frames, mix, target_theta, mix_old, theta_embed=None, pose_embed=None, track=None):
        """A list of PIL / numpy driver frames: every frame is converted, uploaded and queued on its own (four captured frames in
        flight), its uint8 image is produced and copied back on the frame's stream, so the host-side conversions of frame i + 1
        overlap the device work of frame i; the PIL images are wrapped as their copies land.  Same results as one call per frame.
        theta_embed (1,9) / pose_embed (1,E) on the device: the caller's pose / embedding for every frame.  track: the
        frames' poses are smoothed into this PoseTrack (smooth_pose), through the smoothing pipeline."""
        smooth = dict(smooth=True) if track is not None else {}
        pipe = self._driver_pipeline(mix, target_theta, mix_old, theta_embed=theta_embed is not None,
                                     pose_embed=pose_embed is not None, **smooth)
        with_track = (lambda kw: dict(kw, track=track)) if track is not None else (lambda kw: kw)
        return self._render(pipe, len(frames), lambda i: with_track(dict(drv=self._prep(frames[i]), theta_embed=theta_embed,
                                                                         pose_embed=pose_embed)))

    def _pose_track(self) -> PoseTrack:
        """the wrapper's own pose track for smoothed frames in flight, with the wrapper's pose_momentum: its state tensor is
        self.theta, which single smoothed frames carry on, and it is seeded unless tracking was reset (self.theta is None).
        The captured single-frame graph smooths into the same tensor; forward drains the pipeline before it returns, so
        the two paths never overlap."""
        momentum = PoseTrack.check_momentum(self.pose_momentum)
        init = self.theta is None
        tr = self._track
        if init:
            g = self._smooth_graph
            self.theta = g.theta if g is not None else tr.state if tr is not None else \
                torch.zeros((3, 4), dtype=torch.float32, device=self.device)
        if tr is None or tr.state is not self.theta:
            tr = self._track = PoseTrack(self.device, momentum, state=self.theta)
        tr.momentum = momentum
        tr.seeded = not init
        return tr

    def _render(self, pipe, n, inputs):
        """n frames through `pipe`, frame i with the submit arguments inputs(i), returned as forward returns them; sets the
        pred_target_* attributes from the last frame.  A refining pipeline's frames are its refined images, whose uint8
        frames the graph wrote: they are copied straight into the pinned host buffer."""
        from PIL import Image

        refine = getattr(pipe, "refine", None)
        s = self.cfg.image_size if refine is None else refine.cfg.output_size
        img = torch.empty((n, 3, s, s), dtype=torch.float32, device=self.device)
        u8 = torch.empty((n, s, s, 3), dtype=torch.uint8, device=self.device) if refine is None else None
        host = torch.empty((n, s, s, 3), dtype=torch.uint8).pin_memory()
        keep, done = [], []
        for i in range(n):
            kw = inputs(i)
            keep.append(kw)  # read by the slot's stream later: must not return to the allocator (of the current stream) before
            if refine is not None:
                t = pipe.submit(dev_out=img[i:i + 1], u8_out=host[i:i + 1], st=self._state, **kw)
                sl, ev = t.slot, t.done
            else:
                sl = pipe.submit(dev_out=img[i:i + 1], st=self._state, **kw).slot
                with torch.cuda.stream(sl.stream):
                    ops.image_to_u8(img[i:i + 1], out=u8[i:i + 1])  # clamp(0, 1) + ToPILImage (mul(255).byte()) on the device
                    host[i].copy_(u8[i], non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record()
            done.append(ev)
            if len(keep) > 2 * pipe.depth and done[i - 2 * pipe.depth].query():
                keep[i - 2 * pipe.depth] = None
        pred_target_img = []
        for i in range(n):
            done[i].synchronize()
            pred_target_img.append(Image.fromarray(host[i].numpy()))
        pipe.drain()
        so = sl.run.static_state
        self.pred_target_theta = so.pred_target_theta.clone()
        self.pred_target_srt = (so.srt[:, :3].clone(), so.srt[:, 3:6].clone(), so.srt[:, 6:9].clone())
        self.target_pose_embed = so.target_pose_embed.clone()
        return pred_target_img, img

    def _frames(self, driver_images):
        """(n, frame(i) -> (1,3,S,S) on the device): a list of PIL / numpy frames is converted frame by frame, as it is
        queued; anything else (a tensor, one image) at once"""
        if isinstance(driver_images, list) and driver_images and not isinstance(driver_images[0], torch.Tensor):
            return len(driver_images), lambda i: self._prep(driver_images[i])
        drv = self._prep(driver_images)
        return drv.shape[0], lambda i: drv[i:i + 1]

    @torch.no_grad()
    def encode(self, driver_images, mix=False, target_theta=True, mix_old=True):
        """The pose and the expression embedding of every driver frame: the first half of a driver frame (head-pose
        regressor, pose algebra, expression encoder), captured, four frames in flight.  Returns (theta_embed, pose_embed):
        theta_embed = (scale, rotation, translation), each (N,3), the form custome_target_theta_embed takes and
        pred_target_srt has; pose_embed (N,E).  animate(theta_embed, pose_embed) with the same pose options renders the
        frames forward(None, driver_images) renders.
        The expression encoder reads the face aligned by the frame's *mixed* pose (infer.py:568-601), so pose_embed depends
        on mix / mix_old and, with mix=True, on the current identity's source pose: encode with the options and the identity
        the embeddings will be rendered with.  theta_embed is the regressed pose, independent of both; target_theta only
        chooses the rendering warp and has no effect here."""
        if self._state is None:
            raise RuntimeError("encode() called before a source image was given")
        n, frame = self._frames(driver_images)
        pipe = self._driver_pipeline(mix, True, mix_old, encode=True)
        srt = torch.empty((n, 9), dtype=torch.float32, device=self.device)
        pose_embed = torch.empty((n, self.cfg.expr_channels), dtype=torch.float32, device=self.device)
        keep = []
        for i in range(n):
            t = frame(i)
            sl = pipe.submit(t, st=self._state).slot
            so = sl.run.static_state
            with torch.cuda.stream(sl.stream):
                srt[i:i + 1].copy_(so.srt, non_blocking=True)
                pose_embed[i:i + 1].copy_(so.target_pose_embed, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
            keep.append((t, ev))  # t is read by the slot's stream: kept from the allocator until the frame is done (see _render)
            if i >= 2 * pipe.depth and keep[i - 2 * pipe.depth][1].query():
                keep[i - 2 * pipe.depth] = None
        pipe.drain()
        return tuple(srt[:, k:k + 3].contiguous() for k in (0, 3, 6)), pose_embed

    @torch.no_grad()
    def animate(self, theta_embed, pose_embed, mix=False, target_theta=True, mix_old=True):
        """Render N frames of the current identity from N poses and N expression embeddings, with no driver image:
        theta_embed = (scale, rotation, translation), each (N,3) (encode's output, pred_target_srt's form), pose_embed (N,E).
        Captured image-free frames (no head-pose regressor, no expression encoder), four in flight.  Returns
        (list[PIL], img (N,3,H,W)) like forward and sets pred_target_theta, pred_target_srt (the supplied pose) and
        target_pose_embed of the last frame.  Mismatched shapes raise ValueError, no source pass yet RuntimeError, before
        anything is queued."""
        E = self.cfg.expr_channels
        if not isinstance(theta_embed, (tuple, list)) or len(theta_embed) != 3:
            raise ValueError("theta_embed must be (scale, rotation, translation), each (N,3)")
        parts = [torch.as_tensor(t) for t in theta_embed]
        pose_embed = torch.as_tensor(pose_embed)
        if pose_embed.dim() != 2 or pose_embed.shape[1] != E or pose_embed.shape[0] < 1:
            raise ValueError(f"pose_embed must be (N,{E}) with N >= 1, got {tuple(pose_embed.shape)}")
        n = pose_embed.shape[0]
        if any(tuple(p.shape) != (n, 3) for p in parts):
            raise ValueError(f"theta_embed must be three (N,3) tensors with N = {n} (pose_embed's), got "
                             f"{[tuple(p.shape) for p in parts]}")
        if self._state is None:
            raise RuntimeError("animate() called before a source image was given")
        srt = torch.cat([p.to(self.device).float() for p in parts], 1).contiguous()
        pose_embed = pose_embed.to(self.device).float().contiguous()
        pipe = self._driver_pipeline(mix, target_theta, mix_old, image=False, theta_embed=True, pose_embed=True)
        return self._render(pipe, n, lambda i: dict(drv=None, theta_embed=srt[i:i + 1], pose_embed=pose_embed[i:i + 1]))

    @staticmethod
    def _theta_rows(theta_embed) -> torch.Tensor:
        """(scale, rotation, translation), each (N,3), as one (N,9) tensor (ValueError otherwise)"""
        if not isinstance(theta_embed, (tuple, list)) or len(theta_embed) != 3:
            raise ValueError("theta_embed must be (scale, rotation, translation), each (N,3)")
        parts = [torch.as_tensor(t).float() for t in theta_embed]
        if any(p.dim() != 2 or p.shape[1] != 3 or p.shape[0] != parts[0].shape[0] for p in parts) or parts[0].shape[0] < 1:
            raise ValueError(f"theta_embed must be three (N,3) tensors with one N >= 1, got {[tuple(p.shape) for p in parts]}")
        return torch.cat([p.cpu() for p in parts], 1)

    @torch.no_grad()
    def forward_refined(self, driver_images, inferer_s2, mix=False, target_theta=True, mix_old=True,
                        custome_target_theta_embed=None, custome_target_pose_embed=None, bg=None, mask_fn=None):
        """Driver frames refined by stage 2, each in one captured graph: the stage-1 frame, then inferer_s2's stage 2
        (a stage2.InferenceWrapper on this device) on its image, REFINE_DEPTH frames in flight.  Stage 2 runs with the masks
        of the networks plugged into inferer_s2 (modnet, face_idt, and its cloth setting), or unmasked without them.
        bg (3,H,W) + mask_fn (img (1,3,H,W) -> (1,1,H,W), e.g. masks.face_matte): every stage-1 image is composited over bg
        first, as video.connect_img_and_bg does.  The networks run inside the captured frames (INTEGRATION.md "Mask networks in
        captured frames"); a capture they break raises RuntimeError before any frame is queued.
        The refining pipeline is cached with the others (PIPELINES), keyed by the stage-2 model and its precision, the mask
        network objects, cloth and mask_fn.
        driver_images: what forward's driver path takes (a list of PIL / numpy frames, converted as each is queued; a tensor
        batch; one image), with custome_target_theta_embed / custome_target_pose_embed as in forward (one pose / embedding
        for every frame).  driver_images=None with both embeddings: frames rendered from them as animate renders them,
        theta_embed (N,3) x 3 and pose_embed (N,E).  Returns (list[PIL] of the refined S2 x S2 frames, img (N,3,S2,S2) on
        the device); frame i is inferer_s2.forward(x)[2][0] with x = self.forward(None, frame_i, ...)[1], composited as
        video.connect_img_and_bg(x, bg, mask_fn(x)) when bg and mask_fn are given.  Sets pred_target_theta,
        pred_target_srt and target_pose_embed of the last frame.  There is no smooth_pose form: smoothing is a recurrence
        over the frames, which this path does not run.  Refused before anything is queued: no source pass yet
        (RuntimeError), a stage-2 wrapper on another device, mask networks or inputs that do not fit (ValueError)."""
        if self._state is None:
            raise RuntimeError("forward_refined() called before a source image was given")
        s2, extra, bg = self._refining_options(inferer_s2, bg, mask_fn)
        with_bg = (lambda kw: dict(kw, bg=bg)) if bg is not None else (lambda kw: kw)
        E = self.cfg.expr_channels
        if driver_images is None:
            if custome_target_theta_embed is None or custome_target_pose_embed is None:
                raise ValueError("forward_refined(None, ...) renders from custome_target_theta_embed and custome_target_pose_embed: "
                                 "give both, or driver images")
            srt = self._theta_rows(custome_target_theta_embed)
            pe = torch.as_tensor(custome_target_pose_embed).float()
            if pe.dim() != 2 or tuple(pe.shape) != (srt.shape[0], E):
                raise ValueError(f"custome_target_pose_embed must be ({srt.shape[0]},{E}) (one row per pose), got {tuple(pe.shape)}")
            srt, pe = srt.to(self.device).contiguous(), pe.to(self.device).contiguous()
            pipe = self._driver_pipeline(mix, target_theta, mix_old, refine=s2, **extra, image=False, theta_embed=True, pose_embed=True)
            return self._render(pipe, srt.shape[0],
                                lambda i: with_bg(dict(drv=None, theta_embed=srt[i:i + 1], pose_embed=pe[i:i + 1])))
        if isinstance(driver_images, list) and not driver_images:
            raise ValueError("forward_refined: no driver frame")
        srt = pe = None
        if custome_target_theta_embed is not None:
            srt = self._theta_rows(custome_target_theta_embed)
            if srt.shape[0] != 1:
                raise ValueError("with driver images custome_target_theta_embed is one pose (1,3) x 3 for every frame")
            srt = srt.to(self.device).contiguous()
        if custome_target_pose_embed is not None:
            pe = torch.as_tensor(custome_target_pose_embed).float()
            if pe.numel() != E:
                raise ValueError(f"with driver images custome_target_pose_embed is one embedding of {E} values for every frame, "
                                 f"got {tuple(pe.shape)}")
            pe = pe.to(self.device).reshape(1, E).contiguous()
        n, frame = self._frames(driver_images)
        pipe = self._driver_pipeline(mix, target_theta, mix_old, refine=s2, **extra, theta_embed=srt is not None, pose_embed=pe is not None)
        return self._render(pipe, n, lambda i: with_bg(dict(drv=frame(i), theta_embed=srt, pose_embed=pe)))

    def _refining_options(self, inferer_s2, bg, mask_fn):
        """forward_refined's checks of a stage-2 wrapper, its mask networks and a composite: (the stage-2 model, the
        _driver_pipeline options refine_masks= / composite=, bg as a float32 device tensor or None); ValueError if they do not fit"""
        s2 = getattr(inferer_s2, "model_two", None)
        if s2 is None:
            raise ValueError("inferer_s2 must be a stage2.InferenceWrapper")
        if (bg is None) != (mask_fn is None):
            raise ValueError("bg and mask_fn composite the frames together: give both, or neither")
        extra = {}
        modnet, face_idt = getattr(inferer_s2, "modnet", None), getattr(inferer_s2, "face_idt", None)
        if modnet is not None or face_idt is not None:
            extra["refine_masks"] = dict(modnet=modnet, face_idt=face_idt, cloth=bool(getattr(inferer_s2, "cloth", False)))
        if mask_fn is not None:
            extra["composite"] = mask_fn
            s = self.cfg.image_size
            bg = torch.as_tensor(bg)
            if tuple(bg.shape) != (3, s, s) or not bg.is_floating_point():
                raise ValueError(f"bg must be a floating-point background of shape {(3, s, s)}, got {tuple(bg.shape)} {bg.dtype}")
            bg = bg.to(self.device, torch.float32).contiguous()
        self.model.check_refine(s2, encode=False)
        Model.check_refine_masks(s2, extra.get("refine_masks"), mask_fn)
        return s2, extra, bg

    # -- notebooks/infer.py:229-243
    def convert_to_tensor(self, image):
        """PIL image(s) / numpy uint8 (H,W,C) -> fp32 (N,C,H,W) in [0,1] on the device.  uint8 pixels cross the bus as bytes
        (0.79 MB per 512^2 frame instead of 3.1 MB) and become u / 255 in emo_u8_to_image (= transforms.ToTensor)."""
        if isinstance(image, torch.Tensor):
            t = image if image.dim() == 4 else image[None]
            return t.to(self.device).float()
        items = image if isinstance(image, list) else [image]
        arrs = []
        for img in items:
            a = np.asarray(img)
            arrs.append(a[:, :, None] if a.ndim == 2 else a)
        if all(a.dtype == np.uint8 for a in arrs):
            u8 = torch.from_numpy(np.ascontiguousarray(np.stack(arrs))).to(self.device, non_blocking=True)
            return ops.u8_to_image(u8)
        return torch.stack([torch.from_numpy(np.ascontiguousarray(a)).permute(2, 0, 1).float() for a in arrs]).to(self.device)

    def _prep(self, image):
        t = self.convert_to_tensor(image)[:, :3].contiguous()
        s = self.cfg.image_size
        if t.shape[-2:] != (s, s):
            t = ops.resize_bicubic(t, (s, s))  # pre-processing resize, infer.py:401-402 / :554-555
        return t.contiguous().float()

    def forward(self, source_image=None, driver_image=None, source_mask=None, source_mask_add=0, driver_mask=None,
                crop=True, reset_tracking=False, smooth_pose=False, hard_normalize=False, soft_normalize=False,
                delta_yaw=None, delta_pitch=None, cloth=False, thetas_pass='', theta_n=0, target_theta=True, mix=False,
                mix_old=True, c_source_latent_volume=None, c_target_latent_volume=None, custome_target_pose_embed=None,
                custome_target_theta_embed=None, no_grad_infer=True, modnet_mask=False):
        if crop:
            raise NotImplementedError("crop=True needs the external mediapipe face detector (out of scope); pass crop=False "
                                      "with pre-cropped images, as notebooks/E_emo_infer_video.ipynb does")
        if modnet_mask and self.modnet is None:
            raise NotImplementedError("modnet_mask=True needs the external MODNet network: set wrapper.modnet = <module> "
                                      "(repos/MODNet is a separate checkout, not part of the reference tree)")
        # hard_normalize, soft_normalize, cloth, thetas_pass, theta_n are accepted and unused, exactly as in the reference
        # (infer.py:355-357 declares them; nothing in :358-647 reads them).  driver_mask only travels in the reference's
        # data_dict: the expression embedder is called with use_seg=False (:597) and never multiplies by it.
        self.no_grad_infer = no_grad_infer
        self.target_theta, self.mix, self.mix_old = target_theta, mix, mix_old
        if reset_tracking:
            self.center = self.size = self.theta = self.delta_yaw = self.delta_pitch = None
        if delta_yaw is not None:
            self.delta_yaw = delta_yaw
        if delta_pitch is not None:
            self.delta_pitch = delta_pitch

        if source_image is not None:
            src = self._prep(source_image)
            if src.shape[0] != 1:
                raise ValueError("one source image per call (the reference reshapes the latents with view(1, c, d, s, s), infer.py:483)")
            self.source_image = self.source_image_crop = src
            # infer.py:408-426.  face_idt (the external BiSeNet behind masks.FaceParsing) is optional here: without it the face
            # mask is all ones, which is what the reference computes for a frame the parser labels 'face' everywhere
            face_mask = None
            if self.face_idt is not None:
                face_mask = (self.face_idt.forward(src)[0] > 0.6).float()             # :410-411 (trashhold 0.6)
            modnet_matte = self.get_mask(src) if modnet_mask else None               # :413, before the face mask is applied
            if face_mask is not None:
                src = (src * face_mask).float().contiguous()                          # :417
            mask = source_mask.to(self.device).float() if source_mask is not None else face_mask   # :421
            if modnet_mask:
                mask = modnet_matte                                                   # :422
            if mask is not None and source_mask_add:
                mask = mask.clamp_(max=1, min=0)                                      # :423-424
            self.source_img_mask = mask if mask is not None else torch.ones_like(src[:, :1])
            self.source_img = self.source_img_crop_m = src
            st = self.model.source_pass(src, mask=mask, c_source_latent_volume=c_source_latent_volume,
                                        c_target_latent_volume=c_target_latent_volume)
            st.wrapper_inputs = dict(source_image=self.source_image, source_image_crop=self.source_image_crop,
                                     source_img_mask=self.source_img_mask, source_img=self.source_img,
                                     source_img_crop_m=self.source_img_crop_m)
            self._use_identity(st)  # the captured driver graphs load it on their next frame; nothing is re-captured

        if driver_image is None:
            return None
        if self._state is None:
            raise RuntimeError("forward(driver_image=...) called before a source image was given")
        custom_srt = None
        if custome_target_theta_embed is not None:   # (scale, rotation, translation), each (1,3): infer.py:566-567
            custom_srt = torch.cat([torch.as_tensor(t).float().reshape(1, 3) for t in custome_target_theta_embed], 1)
        # one pose / embedding for every frame of the call; the captured frames read them from buffers of their own
        embeds = dict(theta_embed=None if custom_srt is None else custom_srt.to(self.device).contiguous(),
                      pose_embed=None if custome_target_pose_embed is None else
                      torch.as_tensor(custome_target_pose_embed).to(self.device).float().reshape(1, -1).contiguous())
        # smoothed frames, more than one, with the regressed pose and embedding: in flight too, smoothed by the pose steps of
        # the wrapper's track (DriverPipeline(smooth=True)).  A single smoothed frame keeps its one captured graph below
        smooth_custom = smooth_pose and (custom_srt is not None or custome_target_pose_embed is not None)
        if not smooth_custom and isinstance(driver_image, list) and len(driver_image) > 1 and \
                not isinstance(driver_image[0], torch.Tensor):
            track = self._pose_track() if smooth_pose else None
            return self._forward_list(driver_image, mix, target_theta, mix_old, **embeds, track=track)
        drv = self._prep(driver_image)
        if not smooth_pose or (not smooth_custom and drv.shape[0] > 1):
            # captured driver frames (CUDA graphs), four in flight when a list of frames is given (DriverPipeline); same
            # kernels as the eager pass below.  With a custom pose / embedding the graphs take it as an input; the
            # expression encoder is then not captured, and pred_target_srt stays the regressed pose (infer.py:563-564)
            track = self._pose_track() if smooth_pose else None
            smooth = dict(smooth=True) if track is not None else {}
            with_track = dict(track=track) if track is not None else {}
            pipe = self._driver_pipeline(mix, target_theta, mix_old, **{k: v is not None for k, v in embeds.items()}, **smooth)
            img = torch.empty_like(drv)
            for i in range(drv.shape[0]):
                sl = pipe.submit(drv[i:i + 1], dev_out=img[i:i + 1], st=self._state, **embeds, **with_track).slot
            pipe.drain()
            so = sl.run.static_state
            self.pred_target_theta = so.pred_target_theta.clone()
            self.pred_target_srt = (so.srt[:, :3].clone(), so.srt[:, 3:6].clone(), so.srt[:, 6:9].clone())
            self.target_pose_embed = so.target_pose_embed.clone()
        elif smooth_pose and custom_srt is None and custome_target_pose_embed is None:
            # pose smoothing is a recurrence over the frames (infer.py:571-581): the first frame seeds self.theta eagerly, every
            # further frame replays a captured graph that smooths into the same tensor, one after the other on this stream.
            # A reset seeds the captured graph's own state tensor, and a new identity is loaded into it: neither re-captures
            imgs = []
            for i in range(drv.shape[0]):
                g = self._smooth_graph
                if self.theta is None:
                    self.theta = g.theta if g is not None else torch.zeros((3, 4), dtype=torch.float32, device=self.device)
                    im, _, _, so = self.model.driver_pass(self._state, drv[i:i + 1].contiguous(), mix=mix, target_theta=target_theta,
                                                          mix_old=mix_old, smooth_state=self.theta, smooth_momentum=self.pose_momentum,
                                                          smooth_init=True)
                else:
                    key = (bool(mix), bool(target_theta), bool(mix_old), float(self.pose_momentum))
                    if g is None or g.theta is not self.theta or g.key != key:
                        run = self.model.make_driver_graph(self._state, mix=mix, target_theta=target_theta, mix_old=mix_old,
                                                           smooth_state=self.theta, smooth_momentum=self.pose_momentum)
                        g = self._smooth_graph = SimpleNamespace(run=run, theta=self.theta, key=key)
                    g.run.load(self._state)
                    im, so = g.run(drv[i:i + 1]).clone(), g.run.static_state
                imgs.append(im)
            img = imgs[0] if len(imgs) == 1 else torch.cat(imgs)
            self.pred_target_theta = so.pred_target_theta.clone()
            self.pred_target_srt = (so.srt[:, :3].clone(), so.srt[:, 3:6].clone(), so.srt[:, 6:9].clone())
            self.target_pose_embed = so.target_pose_embed.clone()
        else:
            # smooth_pose with a custom pose or embedding: eager frames.  self.theta is the smoothed (3,4) pose carried from
            # frame to frame (infer.py:571-581); the device kernel seeds it with the first frame's pose and updates it in place
            imgs = []
            for i in range(drv.shape[0]):
                init = self.theta is None
                if init:
                    self.theta = torch.zeros((3, 4), dtype=torch.float32, device=self.device)
                im, deep_f, img_f, so = self.model.driver_pass(self._state, drv[i:i + 1].contiguous(), mix=mix,
                                                               target_theta=target_theta, mix_old=mix_old, custom_srt=custom_srt,
                                                               custom_pose_embed=custome_target_pose_embed,
                                                               smooth_state=self.theta, smooth_momentum=self.pose_momentum,
                                                               smooth_init=init)
                imgs.append(im)
            img = imgs[0] if len(imgs) == 1 else torch.cat(imgs)
            self.pred_target_theta = so.pred_target_theta
            self.pred_target_srt = (so.srt[:, :3], so.srt[:, 3:6], so.srt[:, 6:9])
            self.target_pose_embed = so.target_pose_embed
        from PIL import Image

        host = ops.image_to_u8(img.detach().contiguous()).cpu().numpy()  # clamp(0, 1) + ToPILImage (mul(255).byte()) on the device
        pred_target_img = [Image.fromarray(h) for h in host]
        return pred_target_img, img
