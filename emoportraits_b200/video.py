"""Caller-side video loop of the reference's demo notebook (`notebooks/E_emo_infer_video.ipynb` cells 40-51) on top of the two
drop-in wrappers: read the driving video, animate the source with every frame, composite over a background, refine with
stage 2, write the side-by-side video.

What the notebook does per frame (cell 51): `inferer.forward(None, frame, crop=False, smooth_pose=False, target_theta=True,
mix=True, mix_old=False)` -> `connect_img_and_bg` (cell 41: mask^8 blend over an inpainted background) -> `do_stage_2`
(cell 42) -> optional fixed crop (cell 46).  Here the driver frames go through the captured, frames-in-flight pipeline in
chunks (`InferenceWrapper.forward(None, [frames…])`), the blend is one device kernel (`emo_composite`) and stage 2 runs on
the whole chunk as a batch.

The notebook's mask and background come from networks that are not part of the reference tree (BiSeNet face parsing / MODNet
for the matte, a LaMa TorchScript for the background, RetinaFace for the crop): they are inputs here — `mask_fn(img) ->
(N,1,H,W)` and a background image; without them the frames are returned un-composited, exactly what the notebook's
`img[0][0]` is.
"""
from __future__ import annotations

import os
from collections import deque
from types import SimpleNamespace
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import ops


def get_video_frames_as_images(video_path: str, size: int = 512, max_len: Optional[int] = None) -> List["Image.Image"]:
    """cell 47: every frame of the video as an RGB PIL image resized to size x size (bicubic, as the notebook's to_512)"""
    import cv2  # optional dependency of this caller-side helper only
    from PIL import Image

    cap = cv2.VideoCapture(str(video_path))
    if not cap.isOpened():
        raise FileNotFoundError(video_path)
    frames = []
    while max_len is None or len(frames) < max_len:
        ret, frame = cap.read()
        if not ret:
            break
        frames.append(Image.fromarray(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB)).resize((size, size), Image.BICUBIC))
    cap.release()
    return frames


def connect_img_and_bg(img: torch.Tensor, bg: torch.Tensor, mask: torch.Tensor, threshold: float = 0.3) -> torch.Tensor:
    """cell 41: `mask_sss = where(mask > 0.3, mask, 0) ** 8;  mask_sss * img + (1 - mask_sss) * bg`, on the device.
    img (N,3,H,W), bg (3,H,W), mask (N,1,H,W) fp32."""
    return ops.composite(img.contiguous().float(), mask.contiguous().float(), bg.contiguous().float(), threshold)


def drive_image_with_video(inferer, source, frames: Sequence, inferer_s2=None, bg: Optional[torch.Tensor] = None,
                           mask_fn: Optional[Callable[[torch.Tensor], torch.Tensor]] = None, chunk: int = 16,
                           crop_box: Optional[tuple] = None, in_flight: bool = False):
    """cell 51.  `inferer`: stage-1 InferenceWrapper, `inferer_s2`: stage-2 wrapper or None, `source`: PIL image, `frames`:
    driving frames (PIL).  Returns (list of output PIL images, list of cropped PIL images or None, frames).
    bg (3,H,W) tensor + mask_fn: composite every animated frame over the background (cell 41) before stage 2.
    crop_box = (left, upper, right, lower) on the output: the fixed crop of cell 46 (first-frame face box, computed by the
    caller's face detector).
    Each wrapper runs with the `precision=` it was built with: a stage-2 wrapper built with precision="fast" refines every
    chunk in fast mode, exactly as calling that wrapper on the same chunk would.  A stage-1 wrapper built with
    source_precision="fast" runs the one source pass in fast mode, and every frame reads that cached source volume.
    in_flight=True (needs inferer_s2): every frame runs stage 1, the composite (with bg and mask_fn) and stage 2 with the masks
    of the networks plugged into inferer_s2 in one captured graph, with frames in flight (InferenceWrapper.forward_refined),
    `chunk` frames per call; the fixed crop is applied afterwards.  The default (False) runs stage 2 eagerly on each chunk
    as a batch.  Both paths keep the float images between the steps: the notebook rounds every step to uint8 (PIL) before
    the next, this function does not, on either path."""
    from PIL import Image

    if in_flight and inferer_s2 is None:
        raise ValueError("in_flight=True refines the frames in flight: it needs inferer_s2")
    kw = dict(crop=False, smooth_pose=False, target_theta=True, mix=True, mix_old=False, modnet_mask=False)
    outs: List[Image.Image] = []
    frames = list(frames)
    if not frames:
        return [], None if crop_box is None else [], frames
    inferer.forward(source, None, **kw)                       # source pass once (the notebook folds it into the first call)
    dev = inferer.device
    composite = bg is not None and mask_fn is not None
    if in_flight:
        for i in range(0, len(frames), chunk):
            pil, _ = inferer.forward_refined(frames[i:i + chunk], inferer_s2, mix=True, target_theta=True, mix_old=False,
                                             bg=bg if composite else None, mask_fn=mask_fn if composite else None)
            outs.extend(pil)
    else:
        for i in range(0, len(frames), chunk):
            part = frames[i:i + chunk]
            _, img = inferer.forward(None, part, **kw)            # (n,3,H,W) on the device, frames pipelined in flight
            if composite:
                img = connect_img_and_bg(img, bg.to(dev), mask_fn(img))
            if inferer_s2 is not None:
                _, _, s2, _ = inferer_s2.forward(img)             # batch of n through the refinement encoder/decoder
                outs.extend(s2)
            else:
                outs.extend(Image.fromarray(h) for h in ops.image_to_u8(img.contiguous()).cpu().numpy())
    crops = None
    if crop_box is not None:
        size = outs[0].size
        crops = [o.crop(crop_box).resize(size, Image.BICUBIC) for o in outs]
    return outs, crops, frames


def make_video(source, drivers: Sequence, out_frames: Sequence, path: str, fps: float = 30.0, size: int = 512) -> None:
    """cell 48: source | driver | output side by side, mp4v"""
    import cv2
    from PIL import Image

    video = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), fps, (3 * size, size))
    try:
        src = np.asarray(source.resize((size, size), Image.LANCZOS))[:, :, :3]
        for d, o in zip(drivers, out_frames):
            row = np.concatenate([src, np.asarray(d.resize((size, size), Image.LANCZOS))[:, :, :3],
                                  np.asarray(o.resize((size, size), Image.LANCZOS))[:, :, :3]], axis=1)
            video.write(cv2.cvtColor(row, cv2.COLOR_RGB2BGR))
    finally:
        video.release()


def get_bg(source, inpaint_fn: Callable, mask_fn: Callable[[torch.Tensor], torch.Tensor], size: int = 512, device=None):
    """cell 40 on the device: the inpainted background of `source` (a PIL image).  Returns (bg (3,size,size) fp32 on `device`
    (default: the current CUDA device), bg_img: the inpainter's output as a PIL image at the source's size).
    gt = to_tensor(source)[:3] (a uint8 upload); m = mask_fn(gt) ((1,1,H,W), as the compositing mask_fn: masks.face_matte is the
    notebook's mdnt=False, InferenceWrapper.get_mask its mdnt=True); the mask is (m >= 0.8) dilated by cv2.dilate(ones(21, 21),
    iterations=2) (ops.mask_dilate, radius 20); inpaint_fn(gt, mask) is the caller's LaMa; then ToPILImage (mul(255).byte(),
    ops.image_to_u8) and Pillow BICUBIC to size x size (ops.resample_u8), / 255.
    One deviation: the notebook does not clamp the inpainter's output before ToPILImage, and torch's float-to-uint8 conversion
    of values outside [0, 1] is undefined; here they are clamped."""
    from PIL import Image

    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    a = np.array(source)
    u8 = torch.from_numpy(a[:, :, None] if a.ndim == 2 else a)[None].to(dev)
    gt = ops.u8_to_image(u8)[:, :3].contiguous()
    mask = ops.mask_dilate(mask_fn(gt).float().contiguous(), 0.8, 20)
    out = ops.image_to_u8(inpaint_fn(gt, mask)[:1].float().contiguous())[0]
    bg_img = Image.fromarray(out.cpu().numpy())
    if tuple(out.shape[:2]) != (size, size):
        out = ops.resample_u8(out, (size, size), "bicubic")
    return ops.u8_to_image(out[None])[0], bg_img


# row buffers of render_video per frame in flight: one being written out while the next is filled
RING_PER_SLOT = 2
# frames per batch of the stage-1 path: drive_image_with_video's default chunk, so that mask_fn sees the same batches
STAGE1_CHUNK = 16


def _check_box(crop_box):
    import numbers

    if crop_box is None:
        return None
    box = tuple(crop_box)
    if len(box) != 4 or not all(isinstance(v, numbers.Integral) for v in box) or box[2] <= box[0] or box[3] <= box[1]:
        raise ValueError(f"crop_box must be a non-empty box of integers (left, upper, right, lower), got {crop_box}")
    return tuple(int(v) for v in box)


def render_video(inferer, source, frames, path: str, inferer_s2=None, bg: Optional[torch.Tensor] = None,
                 mask_fn: Optional[Callable[[torch.Tensor], torch.Tensor]] = None, crop_box: Optional[tuple] = None,
                 fps: float = 30.0, size: int = 512) -> int:
    """cells 47, 51 and 48 as one streaming loop on the device: animate the inferer's current identity with every driver frame
    and write the side-by-side mp4 (source | driver | output, size x size each) to `path`.  Returns the number of frames
    written.  The identity is the one of the inferer's last source pass (inferer.forward(source, None, crop=False), which
    drive_image_with_video runs itself) or handle; `source` (a PIL image of any mode) is drawn as the left panel.
    frames: a list of RGB PIL images, or a video path, whose BGR frames are uploaded as they are decoded and resized on the
    device to the RGB size x size frames get_video_frames_as_images makes.  Each frame runs through the captured pipelines
    with mix=True, target_theta=True, mix_old=False: refined in flight by inferer_s2 (as forward_refined, with bg / mask_fn
    composited in the graph), or stage 1 alone (four in flight; with bg / mask_fn composited in batches of STAGE1_CHUNK
    frames, as drive_image_with_video does).  The output panel (crop_box: crop then Pillow BICUBIC back to the output size,
    as drive_image_with_video(crop_box=)), then Pillow LANCZOS to size, and the driver panel are written on the device
    straight into a BGR row; the row is copied into one of RING_PER_SLOT pinned buffers per frame in flight and written when
    its copy lands, in order.  Every row is the one make_video writes for drive_image_with_video's outputs (its `crops` with
    crop_box) on the same inputs, bit for bit.
    Refused before anything is queued: no source pass (RuntimeError), a path that cannot be opened (FileNotFoundError),
    non-RGB driver images, bg without mask_fn or mask_fn without bg, a crop box that is empty or not made of integers
    (ValueError)."""
    import cv2
    from PIL import Image

    if inferer.identity is None:
        raise RuntimeError("render_video animates the inferer's current identity: run inferer.forward(source, None, crop=False) first")
    if (bg is None) != (mask_fn is None):
        raise ValueError("bg and mask_fn composite the frames together: give both, or neither")
    crop_box = _check_box(crop_box)
    dev = inferer.device
    cap = None
    if isinstance(frames, (str, os.PathLike)):
        cap = cv2.VideoCapture(str(frames))
        if not cap.isOpened():
            raise FileNotFoundError(frames)
    else:
        frames = list(frames)
        bad = [i for i, f in enumerate(frames) if getattr(f, "mode", None) != "RGB"]
        if bad:
            raise ValueError(f"driver frames must be RGB PIL images (frame {bad[0]} is not)")
    try:
        if inferer_s2 is not None:
            s2, extra, bg = inferer._refining_options(inferer_s2, bg, mask_fn)
            pipe = inferer._driver_pipeline(True, True, False, refine=s2, **extra, theta_embed=False, pose_embed=False)
        else:
            if bg is not None:
                bg = torch.as_tensor(bg).to(dev).contiguous().float()
            pipe = inferer._driver_pipeline(True, True, False, theta_embed=False, pose_embed=False)
        return _render_rows(inferer, pipe, source, frames if cap is None else _decoded(cap), path, inferer_s2 is not None,
                            bg, mask_fn, crop_box, fps, size)
    finally:
        if cap is not None:
            cap.release()


def _decoded(cap):
    while True:
        ret, frame = cap.read()
        if not ret:
            return
        yield frame


def _render_rows(inferer, pipe, source, frames, path, refined, bg, mask_fn, crop_box, fps, size):
    import cv2
    from PIL import Image

    dev, S, s1 = inferer.device, size, inferer.cfg.image_size
    src = torch.from_numpy(np.ascontiguousarray(np.asarray(source.resize((S, S), Image.LANCZOS))[:, :, 2::-1])).to(dev)
    R = RING_PER_SLOT * pipe.depth
    ring = []
    for _ in range(R):
        row = torch.empty((S, 3 * S, 3), dtype=torch.uint8, device=dev)
        row[:, :S] = src                                             # the source panel, BGR, once per row buffer
        ring.append(SimpleNamespace(row=row, host=torch.empty((S, 3 * S, 3), dtype=torch.uint8).pin_memory(), done=None, keep=None))
    writer = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), fps, (3 * S, S))
    pending = deque()
    n = 0

    def flush_one():
        e = pending.popleft()
        e.done.synchronize()
        writer.write(e.host.numpy())
        e.keep = None

    def emit(i, out_u8, drv, stream, keep):
        """frame i's row from its output (H,W,3) RGB uint8 and driver (RGB) images, on `stream`"""
        e = ring[i % R]
        if len(pending) == R:
            flush_one()
        with torch.cuda.stream(stream):
            o = out_u8
            if crop_box is not None:
                o = ops.resample_u8(o, (o.shape[1], o.shape[0]), "bicubic", crop=crop_box)
            ops.resample_u8(o, (S, S), "lanczos", dst=e.row[:, 2 * S:], dst_bgr=True)
            ops.resample_u8(drv, (S, S), "lanczos", dst=e.row[:, S:2 * S], dst_bgr=True)
            e.host.copy_(e.row, non_blocking=True)
            e.done = torch.cuda.Event()
            e.done.record()
        e.keep = keep                                               # read on `stream`: kept from the allocator until done
        pending.append(e)

    def upload(f):
        """(the RGB driver image on the device, the model input exactly as InferenceWrapper._prep makes it)"""
        if isinstance(f, np.ndarray):                                # a decoded BGR frame: get_video_frames_as_images's frame
            drv = ops.resample_u8(torch.from_numpy(f).to(dev, non_blocking=True), (S, S), "bicubic", src_bgr=True)
        else:
            drv = torch.from_numpy(np.array(f)).to(dev, non_blocking=True)
        x = ops.u8_to_image(drv[None])
        if x.shape[-2:] != (s1, s1):
            x = ops.resize_bicubic(x, (s1, s1))
        return drv, x

    try:
        if refined:
            extra = dict(bg=bg) if bg is not None else {}
            for f in frames:
                drv, x = upload(f)
                t = pipe.submit(x, st=inferer.identity, **extra)
                emit(n, t.slot.run.static_u8[0], drv, t.slot.stream, (drv, x))
                n += 1
        else:
            img = torch.empty((STAGE1_CHUNK, 3, s1, s1), dtype=torch.float32, device=dev)
            batch = []
            it = iter(frames)
            while True:
                for f in it:
                    drv, x = upload(f)
                    pipe.submit(x, dev_out=img[len(batch):len(batch) + 1], st=inferer.identity)
                    batch.append((drv, x))
                    if len(batch) == STAGE1_CHUNK:
                        break
                if not batch:
                    break
                pipe.drain()
                out = img[:len(batch)]
                if bg is not None:
                    out = connect_img_and_bg(out, bg, mask_fn(out))
                u8 = ops.image_to_u8(out.contiguous())
                cur = torch.cuda.current_stream(dev)
                for j, (drv, x) in enumerate(batch):
                    emit(n, u8[j], drv, cur, (drv, x, u8))
                    n += 1
                batch = []
            pipe.drain()
        while pending:
            flush_one()
        if refined:
            pipe.drain()
    finally:
        writer.release()
    return n
