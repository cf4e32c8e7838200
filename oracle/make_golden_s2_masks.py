"""TEST INFRASTRUCTURE ONLY.  Golden fixtures of stage 2 with its mask networks: runs the UNMODIFIED reference
notebooks/infer_s2.py InferenceWrapper.forward (:351-376) in this container, with the seeded stand-in networks of
oracle/stub_nets.py plugged in where the external checkouts would be (StubMODNet as `modnet`, the reference FaceParsing over
StubBiSeNet as `face_idt`, as oracle/make_golden_masks.py plugs them into notebooks/infer.py), batch 1, cloth False and True:

    python -m oracle.make_golden_s2_masks 512     # writes tests/golden/s2_masks_512{,_cloth}.pt
    python -m oracle.make_golden_s2_masks 1024    # writes tests/golden/s2_masks_1024{,_cloth}.pt

Records sub-sampled taps: the matte of the resized image, the face mask, the masked residual `add` and the uint8 ffhq frame."""
from __future__ import annotations

import pathlib
import sys

import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
GOLD = ROOT / "tests" / "golden"


def run(output_size: int = 512, cloth: bool = False):
    import numpy as np

    import oracle.ref_harness as H
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2
    from oracle import frames as FR
    from oracle.make_golden import sub
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    w, _, _ = H.build_reference_stage2(output_size, 0)
    sys.modules["repos.face_par_off.model"].BiSeNet = StubBiSeNet
    from networks.volumetric_avatar.face_parcing import FaceParsing  # the reference class, unmodified

    w.model_two.load_state_dict(synthetic_state_dict_s2(Stage2Config(output_size=output_size), 0), strict=True)
    w.model_two.eval()
    w.modnet = StubMODNet()
    w.face_idt = FaceParsing(None, device="cpu", project_dir=str(ROOT))
    w.cloth = cloth
    taps = {}
    orig_get_mask = w.get_mask

    def get_mask(img):   # the reference's own get_mask, recording its second call (on the resized image)
        m = orig_get_mask(img)
        taps.setdefault("mattes", []).append(m.detach().clone())
        return m

    w.get_mask = get_mask
    orig_face = w.face_idt.forward
    w.face_idt.forward = lambda x: taps.setdefault("face", orig_face(x))
    h = w.model_two.decoder.register_forward_hook(lambda m, i, o: taps.__setitem__("add", o[0].detach().clone()))
    seed = 60
    img = FR.frame(256, seed, "smooth")
    with torch.no_grad():
        _, _, pil_ffhq, pred_mask = w.forward(img)
    h.remove()
    matte, face = taps["mattes"][1], taps["face"][0]
    fm = matte if cloth else matte * face
    ffhq8 = torch.from_numpy(np.stack([np.asarray(p) for p in pil_ffhq]).astype(np.float32))
    out = {"output_size": output_size, "seed": seed, "input_size": 256, "cloth": cloth,
           "pred_mask_s8": pred_mask[:, :, ::8, ::8].clone(),
           "matte": sub(matte, 40000), "face_packed": np.packbits(face.numpy().astype(np.uint8)), "face_shape": tuple(face.shape),
           "add": sub(taps["add"] * fm, 60000), "ffhq_uint8": sub(ffhq8, 60000)}
    name = f"s2_masks_{output_size}{'_cloth' if cloth else ''}.pt"
    torch.save(out, GOLD / name)
    print(f"[golden s2 masks {output_size} cloth={cloth}] face mean {face.float().mean().item():.3f} matte mean "
          f"{matte.mean().item():.3f} bytes {(GOLD / name).stat().st_size}")


if __name__ == "__main__":
    size = int(sys.argv[1]) if len(sys.argv) > 1 else 512   # read first: building the reference wrapper resets sys.argv
    for cloth in (False, True):
        run(size, cloth)
