"""Mask pre/post-processing around the EXTERNAL mask networks (SURVEY.md §8f rank 3), on the device.

The reference's face-parsing (BiSeNet, `repos/face_par_off`) and matting (MODNet, `repos/MODNet`) networks are separate
checkouts with downloaded weights; neither is part of the reference tree, so there is no source to restate.  What the tree does
around them is here, with the network supplied by the caller (any callable with the reference's call signature):

  FaceParsing            networks/volumetric_avatar/face_parcing.py:9-81 (same ctor arguments + `net=`; `forward` returns the same
                         four int64 masks)
  modnet_get_mask        notebooks/infer.py:649-684 (InferenceWrapper.get_mask)
  face_matte             notebooks/E_emo_infer_video.ipynb cell 13 (get_mask_fp): the video loop's compositing matte

Normalisation, both bilinear resizes, argmax, label-set membership and the two 'area' resizes are csrc/masks.cu kernels; the
network in the middle runs as whatever the caller supplies (torch module on the same device)."""
from __future__ import annotations

import os
import sys

import torch

from . import ops

PARSING_MEAN = (0.485, 0.456, 0.406)   # face_parcing.py:31
PARSING_STD = (0.229, 0.224, 0.225)    # face_parcing.py:32
# face_parcing.py:37-42 (mask_type None): mask, face_body, mask_body, mask_cloth
_LABELS_DEFAULT = ([1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 7, 8, 9, 14, 17, 18], [1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 7, 8, 9, 17, 18], [18], [16])


class FaceParsing(object):
    def __init__(self, mask_type, device="cuda", project_dir=None, net=None):
        """net: the parsing network (x (N,3,512,512) normalised -> tuple whose first element is (N,19,512,512) logits).  When it is
        None the reference's construction is attempted (face_parcing.py:19-29: BiSeNet from <project_dir>/repos/face_par_off with
        res/cp/79999_iter.pth); without that checkout this raises."""
        if mask_type is not None:
            # the reference only defines face_labels / body_labels / cloth_labels for mask_type None (:40-42) and its forward
            # (:69-79) raises AttributeError for every other value; there is no behaviour to mirror
            raise AttributeError("FaceParsing: mask_type must be None (the reference's forward() fails for any other value: "
                                 "'FaceParsing' object has no attribute 'body_labels', face_parcing.py:70)")
        self.device = torch.device(device)
        if net is None:
            if project_dir is None:
                raise ValueError("FaceParsing needs net= (the external BiSeNet) or project_dir= pointing at a tree with repos/face_par_off")
            path = f"{project_dir}/repos/face_par_off"
            sys.path.append(path)
            sys.path.append(project_dir)
            try:
                from repos.face_par_off.model import BiSeNet  # external checkout, not part of the reference tree
            except ImportError as e:
                raise ImportError(f"FaceParsing: {path} (external face-parsing checkout) is not importable; pass net=") from e
            net = BiSeNet(n_classes=19).to(self.device)
            net.load_state_dict(torch.load(os.path.join(f"{path}/res/cp/79999_iter.pth"), map_location="cpu"))
            net.eval()
        self.net = net
        self.mean = torch.tensor(PARSING_MEAN, dtype=torch.float32, device=self.device)
        self.std = torch.tensor(PARSING_STD, dtype=torch.float32, device=self.device)
        self.mask_labels, self.face_labels, self.body_labels, self.cloth_labels = _LABELS_DEFAULT

    @torch.no_grad()
    def label_masks(self, x):
        """forward's four masks as one uint8 (4,N,1,h,w) tensor of 0 / 1, not widened to int64: what a captured frame keeps."""
        h, w = x.shape[2:]
        x512 = ops.parsing_prepare(x.to(self.device).float().contiguous(), self.mean, self.std, (512, 512))   # :57-58
        y = self.net(x512)[0]                                                                                # :59
        m = ops.parsing_masks(y.float().contiguous(), (h, w), (self.mask_labels, self.face_labels, self.body_labels, self.cloth_labels))
        return m

    @torch.no_grad()
    def forward(self, x):
        """x (N,3,h,w) fp32 in [0,1] on the device -> (mask, face_body, mask_body, mask_cloth), int64 (N,1,h,w) like the reference."""
        m = self.label_masks(x).to(torch.int64)                                                              # zeros_like(labels): int64
        return m[0], m[1], m[2], m[3]

    __call__ = forward


@torch.no_grad()
def modnet_get_mask(modnet, img):
    """notebooks/infer.py:649-684.  img (N,3,h,w) fp32 in [0,1] on the device; modnet(im, True) -> (_, _, matte).  Returns the matte
    (N,1,h,w) at the image's resolution."""
    ref_size = 512
    im_b, im_c, im_h, im_w = img.shape
    if max(im_h, im_w) < ref_size or min(im_h, im_w) > ref_size:
        if im_w >= im_h:
            im_rh = ref_size
            im_rw = int(im_w / im_h * ref_size)
        else:
            im_rw = ref_size
            im_rh = int(im_h / im_w * ref_size)
    else:
        im_rh, im_rw = im_h, im_w
    im_rw = im_rw - im_rw % 32
    im_rh = im_rh - im_rh % 32
    # Normalize((0.5,)*3, (0.5,)*3) (:651-657) is (x - 0.5) / 0.5 = 2x - 1 exactly in fp32: fused into the area resize
    im = ops.resize_area(img.float().contiguous(), (im_rh, im_rw), scale=2.0, shift=-1.0)
    _, _, matte = modnet(im, True)
    return ops.resize_area(matte.float().contiguous(), (im_h, im_w))


def face_matte(face_idt, modnet):
    """The video loop's compositing matte, E_emo_infer_video.ipynb cell 13 (get_mask_fp), as a callable img (N,3,h,w) ->
    (N,1,h,w) fp32 usable as video.drive_image_with_video's / forward_refined's mask_fn: the face-parsing mask (> 0.6) times
    the MODNet matte clamped to [0, 1].  face_idt: a FaceParsing; modnet: the matting network.  It issues no host sync, so a
    captured frame may run it (INTEGRATION.md "Mask networks in captured frames")."""

    @torch.no_grad()
    def mask_fn(img):
        face = (face_idt.forward(img)[0] > 0.6).float()
        return face * modnet_get_mask(modnet, img).clamp_(max=1, min=0)

    return mask_fn
