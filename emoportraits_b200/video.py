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
