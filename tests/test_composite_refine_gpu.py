"""Composited, masked refined frames on the GPU: emo_s2_prepare_composite / emo_s2_masked_stem / emo_s2_finish_masked, the
stage-2 wrapper with its mask networks plugged in, DriverPipeline(refine_masks=, composite=), InferenceWrapper.forward_refined(
bg=, mask_fn=) and video.drive_image_with_video(in_flight=True), with the stand-in networks of oracle/stub_nets.py.

  * Kernels: each new entry point is bit for bit the eager composition it replaces (ops.composite -> emo_s2_prepare; torch's
    x4 * mask -> ops.stem_pack; torch's resized + add * (matte * face), clamp_, ops.image_to_u8), into guarded buffers, at the
    KERNEL_SHAPES of tests/test_refine_stream_gpu.py, with mattes on both sides of the threshold, NaN residuals and cloth; and
    each is held against float64 at the resampler bar.
  * Wrapper: stage2.InferenceWrapper.forward with the stand-in networks against the unmodified reference's fixtures
    (tests/golden/s2_masks_*.pt, oracle/make_golden_s2_masks.py): the matte within test_masks.py's bar, face labels differing
    on fewer than 2e-3 of pixels, the uint8 frame within one level wherever the face masks agree.
  * Pipeline: every composited, masked refined frame bit-identical to the eager per-frame composition, exact and fast, four
    in flight with interleaved identities and a background change, and the image-free input set.
  * Video: drive_image_with_video(in_flight=True) against the chunked path, within one level wherever the two paths' masks
    agree (the stand-in networks run at batch 16 on one path and batch 1 on the other: labels may flip where classes tie).
  * Launch coverage: a composited, masked refined frame's live launches fall in the tested launch tables and listed patterns,
    and the new kernels run at shapes the kernel tests check."""
import gc
import pathlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import model_conv_launches as MCL
import model_op_launches as MOL
import test_model_op_launches_gpu as TMO
import test_op_cases_gpu as TOG
from oracle import frames as FR
from test_refine_stream_gpu import (BASE, KERNEL_SHAPES, N, _context, _guarded, _match, _prepare, _s2_wrapper, _stage2,
                                    _u8_match, _untouched, _wrapper)

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
TOL = TOG.TOL
THR = 0.3


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nets():
    from emoportraits_b200 import masks
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    return StubMODNet().cuda(), masks.FaceParsing(None, device="cuda", net=StubBiSeNet().cuda())


def _matte_like(shape, g):
    """a matte with values on both sides of the threshold, and exactly at it"""
    m = torch.rand(shape, generator=g, device="cuda")
    m.view(-1)[::101] = THR
    return m


# ---- kernels ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,h,w,S", KERNEL_SHAPES)
def test_prepare_composite_matches_composite_then_prepare(n, h, w, S):
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(h * 5 + S + n)
    img = torch.rand((n, 3, h, w), generator=g, device="cuda")
    matte, bg = _matte_like((n, 1, h, w), g), torch.rand((3, h, w), generator=g, device="cuda")
    comp = ops.composite(img, matte, bg, THR)
    thr = torch.tensor(THR, dtype=torch.float32).item()                 # the threshold the kernels compare with
    m = torch.where(matte.double() > thr, matte.double(), 0.0) ** 8
    ref = F.interpolate(m * img.double() + (1 - m) * bg.double(), size=(S, S), mode="bilinear", align_corners=False)
    tol = TOL if S % h == 0 and S % w == 0 else TMO.AFFINE2D_TOL
    for stem in ("none", "exact", "fast"):
        want_resized, want_op, _ = _prepare(comp, S, stem == "fast")
        resized, g0 = _guarded((n, 3, S, S), torch.float32)
        op = guard = None
        args = (None, None, 0.0)
        if stem == "fast":
            op, guard = _guarded((n, 1, S, S, 32), torch.float16)
            args = (None, op.data_ptr(), 16.0)
        elif stem == "exact":
            op, guard = _guarded((n, 1, S, S, 4), torch.float32)
            args = (op.data_ptr(), None, 0.0)
        L.call("emo_s2_prepare_composite", img.data_ptr(), matte.data_ptr(), bg.data_ptr(), THR, n, h, w, S, resized.data_ptr(),
               *args, _stream())
        torch.cuda.synchronize()
        assert _untouched(g0) and (guard is None or _untouched(guard)), "write past the end"
        assert torch.equal(TOG._bits(resized), TOG._bits(want_resized)), (stem, "resized differs from composite -> s2_prepare")
        if op is not None:
            assert torch.equal(op.view(torch.int16 if stem == "fast" else torch.int32),
                               want_op.view(torch.int16 if stem == "fast" else torch.int32)), (stem, "stem operand differs")
        e = (resized.double() - ref).abs().max().item()
        assert e < tol * max(1.0, ref.abs().max().item()), e
    # the ops wrapper
    r2, op2 = ops.s2_prepare_composite(img, matte, bg, S, None, THR)
    assert op2 is None and torch.equal(TOG._bits(r2), TOG._bits(want_resized))


@pytest.mark.parametrize("n,S", sorted({(n, S) for n, _, _, S in KERNEL_SHAPES}))
def test_masked_stem_matches_torch(n, S):
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(S * 3 + n)
    resized = torch.rand((n, 3, S, S), generator=g, device="cuda")
    matte = _matte_like((n, 1, S, S), g)
    x4 = torch.zeros((n, 1, S, S, 4), device="cuda")
    x4[..., :3] = resized.permute(0, 2, 3, 1)[:, None]
    want = (x4 * matte.permute(0, 2, 3, 1)[:, None]).contiguous()          # Stage2Model.forward's masked input
    want_plane = ops.stem_pack(want).hi
    out, g0 = _guarded((n, 1, S, S, 4), torch.float32)
    L.call("emo_s2_masked_stem", resized.data_ptr(), matte.data_ptr(), n, S, out.data_ptr(), None, 0.0, _stream())
    plane, g1 = _guarded((n, 1, S, S, 32), torch.float16)
    L.call("emo_s2_masked_stem", resized.data_ptr(), matte.data_ptr(), n, S, None, plane.data_ptr(), 16.0, _stream())
    torch.cuda.synchronize()
    assert _untouched(g0) and _untouched(g1), "write past the end"
    assert torch.equal(TOG._bits(out), TOG._bits(want)), "not torch's x4 * mask"
    assert torch.equal(plane.view(torch.int16), want_plane.view(torch.int16)), "not stem_pack of it"
    ref = x4.double() * matte.double().permute(0, 2, 3, 1)[:, None]
    assert (out.double() - ref).abs().max().item() < TOL
    rel, ab = TOG.PLANE_BOUND["fp16x1"]
    assert ((plane[..., 12:16].double() - 16 * ref).abs() - rel * 16 * ref.abs() - ab).max().item() <= TOL * 16
    # the ops wrapper, fresh and in place
    assert torch.equal(TOG._bits(ops.s2_masked_stem(resized, matte, False)), TOG._bits(want))
    sp = ops.s2_masked_stem(resized, matte, True)
    assert torch.equal(ops.s2_masked_stem(resized, matte, True, out=sp).hi.view(torch.int16), want_plane.view(torch.int16))


@pytest.mark.parametrize("cloth", [False, True])
@pytest.mark.parametrize("n,S", [(1, 1024), (2, 512), (1, 517)])
def test_finish_masked_matches_torch(n, S, cloth):
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(S + n + 11 * cloth)
    resized = torch.rand((n, 3, S, S), generator=g, device="cuda")
    add = torch.randn((n, 3, S, S), generator=g, device="cuda") * 0.4
    add.view(-1)[::7919] = float("nan")
    matte = _matte_like((n, 1, S, S), g)
    face = (torch.rand((n, 1, S, S), generator=g, device="cuda") > 0.3).to(torch.uint8)
    fm = matte if cloth else matte * face.long().float()
    want = (resized + add * fm).clamp_(min=0, max=1)
    want_u8 = ops.image_to_u8(want)
    out, g0 = _guarded((n, 3, S, S), torch.float32)
    u8, g1 = _guarded((n, S, S, 3), torch.uint8)
    L.call("emo_s2_finish_masked", resized.data_ptr(), add.data_ptr(), matte.data_ptr(), None if cloth else face.data_ptr(), n, S, S,
           out.data_ptr(), u8.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert _untouched(g0) and _untouched(g1), "write past the end"
    assert torch.equal(TOG._bits(out), TOG._bits(want)), "not (resized + add * fm).clamp_(0, 1)"
    assert torch.equal(u8, want_u8), "not image_to_u8 of it"
    assert torch.isnan(out).any()                                       # a NaN stays NaN
    ok = ~torch.isnan(add)
    y = (resized.double() + add.double() * fm.double()).clamp(0, 1)
    assert (out.double() - y)[ok].abs().max().item() < TOL
    y8 = (y * 255).floor().permute(0, 2, 3, 1)
    assert (u8.double() - y8)[ok.permute(0, 2, 3, 1)].abs().max().item() <= 1
    o2, u2 = ops.s2_finish_masked(resized, add, matte, None if cloth else face)
    assert torch.equal(TOG._bits(o2), TOG._bits(want)) and torch.equal(u2, want_u8)


# ---- the stage-2 wrapper against the reference ----------------------------------------------------------------------------
def _s2_wrapper_at(root, size, precision="exact"):
    from emoportraits_b200.stage2 import InferenceWrapper, Stage2Config, synthetic_state_dict_s2

    exp = root / "logs_s2" / f"exp{size}"
    if not exp.exists():
        (exp / "checkpoints").mkdir(parents=True)
        (exp / "args.txt").write_text((GOLD / f"args_s2_{size}.txt").read_text())
        torch.save(synthetic_state_dict_s2(Stage2Config(output_size=size), 0), exp / "checkpoints" / "m.pth")
    return InferenceWrapper(experiment_name=f"exp{size}", model_file_name="m.pth", project_dir=str(root), precision=precision)


@pytest.mark.parametrize("name", ["s2_masks_512", "s2_masks_512_cloth", "s2_masks_1024", "s2_masks_1024_cloth"])
def test_stage2_wrapper_masks_match_reference_fixture(name, tmp_path_factory):
    from emoportraits_b200.masks import modnet_get_mask

    g = torch.load(GOLD / f"{name}.pt", weights_only=False)
    size = g["output_size"]
    s2w = _s2_wrapper_at(tmp_path_factory.mktemp("s2m"), size)
    s2w.modnet, s2w.face_idt = _nets()
    s2w.cloth = g["cloth"]
    img = FR.frame(g["input_size"], g["seed"], "smooth").cuda()
    _, _, pil_ffhq, pred_mask = s2w.forward(img)
    _, resized = s2w.model_two.resize(img)
    matte = modnet_get_mask(s2w.modnet, resized)
    face = s2w.face_idt.forward(resized)[0]
    vals, stride = g["matte"]
    assert (matte.reshape(-1)[::stride].cpu() - vals).abs().max().item() <= 2e-4
    assert (pred_mask[:, :, ::8, ::8] - g["pred_mask_s8"]).abs().max().item() <= 2e-4
    ref_face = torch.from_numpy(np.unpackbits(g["face_packed"])[:int(np.prod(g["face_shape"]))].reshape(g["face_shape"]).astype(np.int64))
    agree = face.cpu() == ref_face
    assert (~agree).float().mean().item() < 2e-3
    vals, stride = g["ffhq_uint8"]
    got = torch.from_numpy(np.asarray(pil_ffhq[0]).astype(np.float32)).reshape(-1)[::stride]
    keep = torch.ones_like(got, dtype=torch.bool) if g["cloth"] else agree[0, 0][..., None].expand(size, size, 3).reshape(-1)[::stride]
    d = (got - vals).abs()[keep]
    print(f"\n[{name}] matte / face agree {agree.float().mean().item():.5f}, ffhq uint8 largest difference {d.max().item():.0f}")
    assert d.max().item() <= 1


# ---- pipeline ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    return _context(256)


def _eager(s2, s1, bg, mask_fn, modnet, face_idt, cloth):
    """the eager per-frame composition: the composite, the reference's stage-2 masks, Stage2Model.forward"""
    from emoportraits_b200 import masks, video

    x = video.connect_img_and_bg(s1, bg, mask_fn(s1))
    _, resized = s2.resize(x)
    matte = masks.modnet_get_mask(modnet, resized)
    face = None if cloth else face_idt.forward(resized)[0]
    return s2.forward(x, matte, face)[2]


def _run(pipe, frames, s2_size):
    from test_refine_stream_gpu import _run as run

    return run(pipe, frames, s2_size)


def _check(s2, got, bgs, mask_fn, modnet, face_idt, cloth=False):
    from emoportraits_b200 import ops

    for k, (ref_img, u8, s1) in enumerate(got):
        ffhq = _eager(s2, s1, bgs[k], mask_fn, modnet, face_idt, cloth)
        assert torch.equal(TOG._bits(ref_img), TOG._bits(ffhq)), f"frame {k}: differs from the eager composition"
        assert torch.equal(u8, ops.image_to_u8(ffhq)), f"frame {k}: uint8 frame differs"


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_four_in_flight_interleaved_identities_and_backgrounds(ctx, precision):
    from emoportraits_b200 import masks
    from emoportraits_b200.infer import DriverPipeline

    s2 = _stage2(512, precision)
    modnet, face_idt = _nets()
    mask_fn = masks.face_matte(*_nets()[::-1])
    bgs = [FR.frame(256, 90 + k, "smooth")[0].cuda() for k in range(2)]
    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=4, refine=s2, refine_masks=dict(modnet=modnet, face_idt=face_idt),
                          composite=mask_fn, **BASE)
    order = "ABBABAAB"
    per_frame = [bgs[0] if k < 3 else bgs[1] for k in range(len(order))]      # the background changes after frame 2
    got = _run(pipe, [dict(drv=ctx.drv[k % N], st=ctx.st[who], bg=per_frame[k]) for k, who in enumerate(order)], 512)
    _check(s2, got, per_frame, mask_fn, modnet, face_idt)
    _match([g[2] for g in got], [ctx.model.driver_pass(ctx.st[who], ctx.drv[k % N], **BASE)[0] for k, who in enumerate(order)])
    assert (got[0][0] - got[1][0]).abs().max().item() > 1e-2


def test_image_free_composited_masked_frames_with_cloth(ctx):
    from emoportraits_b200 import masks
    from emoportraits_b200.infer import DriverPipeline

    s2 = _stage2(512, "fast")
    modnet, face_idt = _nets()
    mask_fn = masks.face_matte(*_nets()[::-1])
    bg = FR.frame(256, 93, "smooth")[0].cuda()
    pipe = DriverPipeline(ctx.model, ctx.st["B"], depth=2, refine=s2, refine_masks=dict(modnet=modnet, face_idt=face_idt, cloth=True),
                          composite=mask_fn, image=False, theta_embed=True, pose_embed=True, **BASE)
    got = _run(pipe, [dict(drv=None, theta_embed=ctx.srt[i], pose_embed=ctx.pe[i], bg=bg) for i in range(N)], 512)
    _check(s2, got, [bg] * N, mask_fn, modnet, face_idt, cloth=True)


def test_flagship_size_512_to_1024():
    from emoportraits_b200 import masks
    from emoportraits_b200.infer import DriverPipeline

    c = _context(512)
    modnet, face_idt = _nets()
    mask_fn = masks.face_matte(*_nets()[::-1])
    bg = FR.frame(512, 94, "smooth")[0].cuda()
    for precision in ("exact", "fast"):
        s2 = _stage2(1024, precision)
        pipe = DriverPipeline(c.model, c.st["A"], depth=2, refine=s2, refine_masks=dict(modnet=modnet, face_idt=face_idt),
                              composite=mask_fn, **BASE)
        got = _run(pipe, [dict(drv=d, bg=bg) for d in c.drv[:3]], 1024)
        _check(s2, got, [bg] * 3, mask_fn, modnet, face_idt)
        del pipe, got
        gc.collect()


# ---- wrapper and video loop ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def s2_root(tmp_path_factory):
    return tmp_path_factory.mktemp("s2c")


def test_forward_refined_composited_matches_two_wrappers(ctx, s2_root):
    from emoportraits_b200 import masks, video

    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    s2w = _s2_wrapper_at(s2_root, 512)
    s2w.modnet, s2w.face_idt = _nets()
    mask_fn = masks.face_matte(*_nets()[::-1])
    bg = FR.frame(256, 95, "smooth")[0].cuda()
    pils = [FR.pil(ctx.size, 50 + i, "smooth") for i in range(N)]
    got, img = w.forward_refined(pils, s2w, bg=bg, mask_fn=mask_fn, **BASE)
    assert len(got) == N and img.shape == (N, 3, 512, 512)
    want = []
    for p in pils:
        x = w.forward(None, p, crop=False, **BASE)[1]
        want.append(s2w.forward(video.connect_img_and_bg(x, bg, mask_fn(x)))[2][0])
    _u8_match(got, want, "composited, masked")
    n_pipes = len(w._pipelines)
    w.forward_refined(pils[:1], s2w, bg=bg, mask_fn=mask_fn, **BASE)          # cached
    assert len(w._pipelines) == n_pipes
    s2w.cloth = True
    w.forward_refined(pils[:1], s2w, bg=bg, mask_fn=mask_fn, **BASE)          # cloth is part of the key
    assert len(w._pipelines) == n_pipes + 1


def test_drive_image_with_video_in_flight_matches_chunked(ctx, s2_root):
    from emoportraits_b200 import masks, video

    w = _wrapper(ctx)
    s2w = _s2_wrapper_at(s2_root, 512)
    modnet, face_idt = _nets()
    s2w.modnet, s2w.face_idt = modnet, face_idt
    mfi, mmod = _nets()[::-1]
    mask_fn = masks.face_matte(mfi, mmod)
    bg = FR.frame(256, 96, "smooth")[0].cuda()
    src = FR.pil(256, 41, "smooth")
    pils = [FR.pil(256, 50 + i, "smooth") for i in range(6)]
    flight, fc, _ = video.drive_image_with_video(w, src, pils, inferer_s2=s2w, bg=bg, mask_fn=mask_fn, crop_box=(64, 64, 448, 448),
                                                in_flight=True)
    chunked, cc, _ = video.drive_image_with_video(w, src, pils, inferer_s2=s2w, bg=bg, mask_fn=mask_fn, crop_box=(64, 64, 448, 448))
    assert len(flight) == len(chunked) == len(fc) == len(cc) == 6
    # where the two paths' masks agree: the stage-2 face labels and the compositing matte of each path's own batching
    s1 = w.forward(None, pils, crop=False, **BASE)[1]
    m16 = mask_fn(s1)
    m1 = torch.cat([mask_fn(s1[i:i + 1]) for i in range(6)])
    x16 = video.connect_img_and_bg(s1, bg, m16)
    x1 = torch.cat([video.connect_img_and_bg(s1[i:i + 1], bg, m1[i:i + 1]) for i in range(6)])
    r16, r1 = s2w.model_two.resize(x16)[1], s2w.model_two.resize(x1)[1]
    f16 = face_idt.forward(r16)[0]
    f1 = torch.cat([face_idt.forward(r1[i:i + 1])[0] for i in range(6)])
    comp_differs = F.interpolate((m16 != m1).float(), size=(512, 512), mode="nearest")
    differs = (F.max_pool2d(comp_differs, 7, 1, 3) > 0) | (f16 != f1) | (modnet_masks_differ(modnet, r16, r1))
    worst, flipped = 0, differs.float().mean().item()
    for k, (a, b) in enumerate(zip(flight, chunked)):
        d = np.abs(np.asarray(a).astype(int) - np.asarray(b).astype(int)).max(axis=2)
        worst = max(worst, int(d[~differs[k, 0].cpu().numpy()].max()))
    print(f"\n[in flight vs chunked] largest difference {worst} level(s) where the masks agree ({flipped:.2e} of pixels differ)")
    assert worst <= 1 and flipped < 2e-2


def modnet_masks_differ(modnet, r16, r1):
    """pixels where the stage-2 matte of the batch-16 and the batch-1 run differ by more than the stand-in's rounding"""
    from emoportraits_b200.masks import modnet_get_mask

    a = modnet_get_mask(modnet, r16)
    b = torch.cat([modnet_get_mask(modnet, r1[i:i + 1]) for i in range(r1.shape[0])])
    return (a - b).abs() > 1e-3


# ---- launch coverage ------------------------------------------------------------------------------------------------------
def test_composited_masked_frame_launches_fall_in_tested_classes(s2_root):
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import masks

    c = _context(256)
    w = _wrapper(c)
    w.forward(c.src["A"], None, crop=False)
    lib = L.load()
    ops_table = {MOL.key(r) for r in MOL.load()}
    conv_table = {MCL.key(r) for r in MCL.load()}
    boundary_ops = {r["op"] for r in MOL.BOUNDARY}
    listed = {MOL.pattern(r) for r in MOL.BOUNDARY}
    handoff = ("emo_s2_prepare_composite", "emo_s2_masked_stem", "emo_s2_finish_masked")
    seen = {"op": [], "conv": [], "boundary": [], "handoff": []}
    launch = L.call

    def call(name, *args):
        if name == "emo_conv_igemm":
            seen["conv"].append(MCL.launch_record(L, lib, args[0]._obj))
        elif name in handoff:
            seen["handoff"].append((name, args))
        elif name[4:] in boundary_ops:
            seen["boundary"].append(MOL.launch_record(name, args))
        elif name not in MOL.NOT_RECORDED:
            seen["op"].append(MOL.launch_record(name, args))
        return launch(name, *args)

    pils = [FR.pil(256, 50 + i, "smooth") for i in range(3)]
    bg = FR.frame(256, 97, "smooth")[0].cuda()
    mp = pytest.MonkeyPatch()
    mp.setattr(L, "call", call)
    try:
        for precision in ("exact", "fast"):
            s2w = _s2_wrapper_at(s2_root, 512, precision)
            s2w.modnet, s2w.face_idt = _nets()
            w.forward_refined(pils, s2w, bg=bg, mask_fn=masks.face_matte(*_nets()[::-1]), **BASE)
        torch.cuda.synchronize()
    finally:
        mp.undo()
    print(f"\n[composited, masked frame launches] {len(seen['op'])} op, {len(seen['conv'])} conv, {len(seen['boundary'])} boundary, "
          f"{len(seen['handoff'])} handoff")
    assert seen["op"] and seen["conv"] and seen["boundary"] and {n for n, _ in seen["handoff"]} == set(handoff)
    assert not [r for r in seen["op"] if MOL.key(r) not in ops_table]
    assert not [r for r in seen["conv"] if MCL.key(r) not in conv_table]
    assert not [r for r in seen["boundary"] if MOL.pattern(r) not in listed]
    tested_prepare = {(h, w_, S) for _, h, w_, S in KERNEL_SHAPES}
    for name, args in seen["handoff"]:
        if name == "emo_s2_prepare_composite":
            assert args[4] in (1, 2) and tuple(args[5:8]) in tested_prepare, args[4:8]
        elif name == "emo_s2_masked_stem":
            assert (args[2], args[3]) in {(n, S) for n, _, _, S in KERNEL_SHAPES}, args[2:4]
        else:
            assert args[4] in (1, 2) and (args[5], args[6]) in {(512, 512), (1024, 1024), (517, 517)}, args[4:7]
