"""Refined frames in flight on the GPU: emo_s2_prepare / emo_s2_finish, DriverPipeline(refine=) and
InferenceWrapper.forward_refined.

  * Kernels: emo_s2_prepare is emo_resize_bilinear -> permute for `resized` and emo_resize_bilinear (-> emo_stem_pack) for the
    stem's operand, bit for bit, at 512 -> 1024 and 256 -> 512 for N = 1 and 2 and at an odd size; emo_s2_finish is torch's
    (resized + add).clamp_(0, 1) followed by ops.image_to_u8, bit for bit.  Outputs start as NaN / 0xA5 with a guard region
    after them: every element is written and nothing past the end.  Both are held against float64 at the resampler bar of
    tests/test_model_op_launches_gpu.py (2e-5 of the scale; the fp16 plane at its format's bound; 1e-4 at the odd size, whose
    fp32 source coordinates are inexact).
  * Pipeline: each refined frame is bit-identical to the eager Stage2Model.forward of the stage-1 image the captured frame
    made (batch 1), exact and fast, at 256^2 -> 512^2 and 512^2 -> 1024^2; four frames in flight with interleaved identities
    and the image-free input set too.  The stage-1 images follow the in-flight rule of DESIGN.md section 2.4 against the
    eager driver pass.
  * Wrapper: forward_refined against the per-frame composition of the two wrappers (uint8 for uint8, in-flight rule), against
    video.drive_image_with_video's chunked stage 2 (batch 16: every pixel within one level), the pipeline cache and the
    errors.
  * Launch coverage: a refined frame's live launches at 256^2 -> 512^2 are entries of the tested launch tables; stage 2 at
    batch 1 @1024^2 (not a configuration of the tables) is recorded in EMO_DRY_RUN mode and every launch not in the tables is
    replayed against float64 with the replay code of tests/test_model_conv_launches_gpu.py / test_model_op_launches_gpu.py."""
import gc
import math
import pathlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import model_conv_launches as MCL
import model_op_launches as MOL
import test_model_conv_launches_gpu as TMC
import test_model_op_launches_gpu as TMO
import test_op_cases_gpu as TOG
from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
GUARD = 4096
TOL = TOG.TOL                 # 2e-5 of max(1, scale): the resampler bar of the launch replay
N = 5
BASE = dict(mix=True, mix_old=False)     # the video loop's options (video.drive_image_with_video)
KERNEL_SHAPES = [(1, 512, 512, 1024), (2, 512, 512, 1024), (1, 256, 256, 512), (2, 256, 256, 512), (1, 300, 260, 517)]


@pytest.fixture(autouse=True)
def _release():
    """collect each test's wrappers and captured graphs here, with no capture in progress (tests/test_embedding_drive_gpu.py)"""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _guarded(shape, dtype):
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), 0xA5 if dtype == torch.uint8 else float("nan"), dtype=dtype, device="cuda")
    return buf[:n].view(shape), buf[n:]


def _untouched(guard):
    return bool((guard == 0xA5).all()) if guard.dtype == torch.uint8 else bool(torch.isnan(guard.float()).all())


def _prepare(img, S, fast):
    """emo_s2_prepare into guarded buffers: (resized, operand, guards)"""
    from emoportraits_b200 import lib as L

    n, _, h, w = img.shape
    resized, g0 = _guarded((n, 3, S, S), torch.float32)
    if fast:
        op, g1 = _guarded((n, 1, S, S, 32), torch.float16)
        args = (None, op.data_ptr(), 16.0)
    else:
        op, g1 = _guarded((n, 1, S, S, 4), torch.float32)
        args = (op.data_ptr(), None, 0.0)
    L.call("emo_s2_prepare", img.data_ptr(), n, h, w, S, resized.data_ptr(), *args, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return resized, op, (g0, g1)


# ---- kernels ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,h,w,S", KERNEL_SHAPES)
def test_prepare_matches_resize_and_stem_pack(n, h, w, S):
    from emoportraits_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(h * 7 + S + n)
    img = torch.rand((n, 3, h, w), generator=g, device="cuda")        # white noise: the largest steps between pixels
    x4 = ops.resize_bilinear(img, (S, S))
    want_resized = x4[:, 0, :, :, :3].permute(0, 3, 1, 2).contiguous()
    want_plane = ops.stem_pack(x4).hi
    ref = F.interpolate(img.double(), size=(S, S), mode="bilinear", align_corners=False)
    scale = img.abs().max().item()
    # the model's ratios (x2) have exact fp32 source coordinates: the resampler bar.  At the odd size (300 / 517) the fp32
    # coordinate itself is inexact, as in emo_resize_bilinear and torch's fp32 kernel: the bar of DESIGN.md section 2 item 5
    tol = TOL if S % h == 0 and S % w == 0 else TMO.AFFINE2D_TOL
    for fast in (False, True):
        resized, op, guards = _prepare(img, S, fast)
        assert all(_untouched(gd) for gd in guards), "write past the end"
        assert torch.equal(TOG._bits(resized), TOG._bits(want_resized)), (fast, "resized")
        if fast:
            assert torch.equal(op.view(torch.int16), want_plane.view(torch.int16)), "fp16 plane differs from stem_pack's"
            # the centre tap (kx = 3) against float64: the fp16 plane's bound of the scaled value
            rel, ab = TOG.PLANE_BOUND["fp16x1"]
            y = ref.permute(0, 2, 3, 1)[:, None] * 16.0
            got = op[..., 12:15].double()
            assert ((got - y).abs() - rel * y.abs() - ab).max().item() <= TOL * 16 * max(1.0, scale)
        else:
            assert torch.equal(TOG._bits(op), TOG._bits(x4)), "x4 differs from resize_bilinear's"
        e = (resized.double() - ref).abs().max().item()
        assert e < tol * max(1.0, scale), e
        print(f"\n[s2_prepare {n}x{h}x{w}->{S} {'fast' if fast else 'exact'}] resized vs float64 {e:.2e}")


@pytest.mark.parametrize("n,S", [(1, 1024), (2, 512), (1, 517)])
def test_finish_matches_torch(n, S):
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(S + n)
    resized = torch.rand((n, 3, S, S), generator=g, device="cuda")
    add = torch.randn((n, 3, S, S), generator=g, device="cuda") * 0.3    # both clamp bounds are reached
    add.view(-1)[::7919] = float("nan")
    want = (resized + add).clamp_(min=0, max=1)
    want_u8 = ops.image_to_u8(want)
    out, g0 = _guarded((n, 3, S, S), torch.float32)
    u8, g1 = _guarded((n, S, S, 3), torch.uint8)
    L.call("emo_s2_finish", resized.data_ptr(), add.data_ptr(), n, S, S, out.data_ptr(), u8.data_ptr(),
           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert _untouched(g0) and _untouched(g1), "write past the end"
    assert torch.equal(TOG._bits(out), TOG._bits(want)), "not (resized + add).clamp_(0, 1)"
    assert torch.equal(u8, want_u8), "not image_to_u8 of it"
    # against float64: the clamped sum, and the byte within one level of trunc(255 y) (a level boundary may fall between them)
    ok = ~torch.isnan(add)
    y = (resized.double() + add.double()).clamp(0, 1)
    assert (out.double() - y)[ok].abs().max().item() < TOL
    y8 = (y * 255).floor().permute(0, 2, 3, 1)
    assert (u8.double() - y8)[ok.permute(0, 2, 3, 1)].abs().max().item() <= 1
    # the same through the ops wrapper
    o2, u2 = ops.s2_finish(resized, add)
    assert torch.equal(TOG._bits(o2), TOG._bits(want)) and torch.equal(u2, want_u8)


# ---- pipeline ---------------------------------------------------------------------------------------------------------------
def _stage2(size, precision, device="cuda"):
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2

    cfg = Stage2Config(output_size=size)
    return Stage2Model(cfg, synthetic_state_dict_s2(cfg, 0), device, precision=precision)


def _context(size):
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    cfg = shipped_config(size)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    model = Model(cfg, sd, hsd, "cuda")
    src = {k: FR.frame(size, s, "smooth").cuda() for k, s in {"A": 41, "B": 61}.items()}
    st = {k: model.source_pass(x) for k, x in src.items()}
    drv = [FR.frame(size, 50 + i, "smooth").cuda() for i in range(N)]
    enc = [model.driver_pass(st["A"], d, mix=True, encode_only=True)[3] for d in drv]
    srt = [enc[(i + 1) % N].srt.clone() for i in range(N)]
    pe = [enc[(i + 2) % N].target_pose_embed.clone() for i in range(N)]
    return SimpleNamespace(size=size, cfg=cfg, sd=sd, hsd=hsd, model=model, src=src, st=st, drv=drv, srt=srt, pe=pe)


@pytest.fixture(scope="module")
def ctx():
    return _context(256)


def _match(got, want, what=""):
    """the in-flight rule (DESIGN.md section 2.4): every frame bit-identical but at most one, and that one within 5e-4"""
    errs = [(g.float().cpu() - w.float().cpu()).abs().max().item() for g, w in zip(got, want)]
    assert len(errs) == len(want) and max(errs) < 5e-4 and sum(e == 0.0 for e in errs) >= len(errs) - 1, (what, errs)


def _run(pipe, frames, s2_size):
    """submit every frame (kw dicts of submit); returns per frame (refined, u8, stage-1 image) copied on the frame's stream"""
    out = []
    for kw in frames:
        s1 = pipe.model.cfg.image_size
        o = (torch.empty((1, 3, s2_size, s2_size), device="cuda"), torch.empty((1, s2_size, s2_size, 3), dtype=torch.uint8, device="cuda"),
             torch.empty((1, 3, s1, s1), device="cuda"))
        t = pipe.submit(dev_out=o[0], u8_out=o[1], **kw)
        with torch.cuda.stream(t.slot.stream):
            o[2].copy_(t.slot.run.static_stage1)
        out.append(o)
    pipe.drain()
    torch.cuda.synchronize()
    return out


def _check_refined(s2, got):
    """each refined frame and its bytes against the eager Stage2Model.forward of its own stage-1 image, bit for bit"""
    from emoportraits_b200 import ops

    for k, (ref_img, u8, s1) in enumerate(got):
        resized, _, ffhq = s2.forward(s1)
        assert torch.equal(TOG._bits(ref_img), TOG._bits(ffhq)), f"frame {k}: refined image differs from the eager stage 2"
        assert torch.equal(u8, ops.image_to_u8(ffhq)), f"frame {k}: uint8 frame differs"


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_refined_frames_match_eager_stage2(ctx, precision):
    from emoportraits_b200.infer import DriverPipeline

    s2 = _stage2(512, precision)
    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=2, refine=s2, **BASE)
    got = _run(pipe, [dict(drv=d) for d in ctx.drv], 512)
    _check_refined(s2, got)
    _match([g[2] for g in got], [ctx.model.driver_pass(ctx.st["A"], d, **BASE)[0] for d in ctx.drv], precision)
    assert pipe.slots[0].run.static_out.shape == (1, 3, 512, 512) and pipe.slots[0].run.static_u8.shape == (1, 512, 512, 3)


def test_four_in_flight_interleaved_identities(ctx):
    from emoportraits_b200.infer import DriverPipeline

    s2 = _stage2(512, "exact")
    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=4, refine=s2, **BASE)
    order = "ABBABAAB"
    got = _run(pipe, [dict(drv=ctx.drv[k % N], st=ctx.st[who]) for k, who in enumerate(order)], 512)
    _check_refined(s2, got)
    _match([g[2] for g in got], [ctx.model.driver_pass(ctx.st[who], ctx.drv[k % N], **BASE)[0] for k, who in enumerate(order)])
    assert (got[0][0] - got[1][0]).abs().max().item() > 1e-2      # the identities differ visibly


def test_image_free_refined_frames(ctx):
    from emoportraits_b200.infer import DriverPipeline

    s2 = _stage2(512, "fast")
    pipe = DriverPipeline(ctx.model, ctx.st["B"], depth=2, refine=s2, image=False, theta_embed=True, pose_embed=True, **BASE)
    got = _run(pipe, [dict(drv=None, theta_embed=ctx.srt[i], pose_embed=ctx.pe[i]) for i in range(N)], 512)
    _check_refined(s2, got)
    _match([g[2] for g in got], [ctx.model.driver_pass(ctx.st["B"], None, custom_srt=ctx.srt[i], custom_pose_embed=ctx.pe[i], **BASE)[0]
                                 for i in range(N)])


def test_flagship_size_512_to_1024():
    from emoportraits_b200.infer import DriverPipeline

    c = _context(512)
    for precision in ("exact", "fast"):
        s2 = _stage2(1024, precision)
        pipe = DriverPipeline(c.model, c.st["A"], depth=2, refine=s2, **BASE)
        got = _run(pipe, [dict(drv=d) for d in c.drv[:3]], 1024)
        _check_refined(s2, got)
        _match([g[2] for g in got], [c.model.driver_pass(c.st["A"], d, **BASE)[0] for d in c.drv[:3]], precision)
        del pipe, got
        gc.collect()


# ---- wrapper ----------------------------------------------------------------------------------------------------------------
def _wrapper(ctx, **kw):
    from emoportraits_b200.infer import InferenceWrapper

    return InferenceWrapper("refine", args_path=GOLD / f"args_{ctx.size}.txt", state_dict=ctx.sd, head_pose_state_dict=ctx.hsd,
                            print_params=False, **kw)


@pytest.fixture(scope="module")
def s2_ckpt(tmp_path_factory):
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2

    root = tmp_path_factory.mktemp("s2")
    ckpt = root / "logs_s2" / "exp" / "checkpoints"
    ckpt.mkdir(parents=True)
    (root / "logs_s2" / "exp" / "args.txt").write_text((GOLD / "args_s2_512.txt").read_text())
    torch.save(synthetic_state_dict_s2(Stage2Config(output_size=512), 0), ckpt / "m.pth")
    return root


def _s2_wrapper(root, precision="exact"):
    from emoportraits_b200.stage2 import InferenceWrapper

    return InferenceWrapper(experiment_name="exp", model_file_name="m.pth", project_dir=str(root), precision=precision)


def _u8_match(got, want, what=""):
    """uint8 frames under the in-flight rule: all equal but at most one frame, that one within one level"""
    diffs = [int(np.abs(np.asarray(g).astype(int) - np.asarray(w).astype(int)).max()) for g, w in zip(got, want)]
    assert len(diffs) == len(want) and max(diffs) <= 1 and sum(d == 0 for d in diffs) >= len(diffs) - 1, (what, diffs)


def test_forward_refined_matches_two_wrappers(ctx, s2_ckpt):
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    s2w = _s2_wrapper(s2_ckpt)
    pils = [FR.pil(ctx.size, 50 + i, "smooth") for i in range(N)]
    got, img = w.forward_refined(pils, s2w, **BASE)
    assert len(got) == N and img.shape == (N, 3, 512, 512) and got[0].size == (512, 512)
    want = [s2w.forward(w.forward(None, p, crop=False, **BASE)[1])[2][0] for p in pils]
    _u8_match(got, want, "two wrappers")
    # the device images are the refined frames the PIL images were made from
    assert all(np.array_equal(np.asarray(g), h) for g, h in zip(got, ops_u8(img)))
    # against the chunked path: stage 2 at batch 16 after a captured stage-1 list
    from emoportraits_b200 import video

    chunked, _, _ = video.drive_image_with_video(w, ctx.src["A"], pils, inferer_s2=s2w, chunk=16)
    worst = max(int(np.abs(np.asarray(g).astype(int) - np.asarray(c).astype(int)).max()) for g, c in zip(got, chunked))
    print(f"\n[forward_refined vs drive_image_with_video chunk 16] largest difference {worst} level(s)")
    assert worst <= 1


def ops_u8(img):
    from emoportraits_b200 import ops

    return ops.image_to_u8(img.contiguous()).cpu().numpy()


def test_forward_refined_inputs_and_cache(ctx, s2_ckpt):
    w = _wrapper(ctx)
    w.forward(ctx.src["B"], None, crop=False)
    s2w, s2f = _s2_wrapper(s2_ckpt), _s2_wrapper(s2_ckpt, precision="fast")
    # a tensor batch, one image, and the image-free form against the per-frame composition
    batch = torch.cat(ctx.drv[:3])
    got, _ = w.forward_refined(batch, s2f, **BASE)
    _u8_match(got, [s2f.forward(w.forward(None, ctx.drv[i], crop=False, **BASE)[1])[2][0] for i in range(3)], "batch")
    one, _ = w.forward_refined(ctx.drv[0], s2f, **BASE)
    assert len(one) == 1
    pipe = next(reversed(w._pipelines.values()))
    assert pipe.refine is s2f.model_two and pipe.depth == w.REFINE_DEPTH
    n_pipes = len(w._pipelines)
    w.forward_refined(ctx.drv[1], s2f, **BASE)                      # cached: no new pipeline
    assert len(w._pipelines) == n_pipes and next(reversed(w._pipelines.values())) is pipe
    theta = tuple(torch.cat([s[:, k:k + 3] for s in ctx.srt]) for k in (0, 3, 6))
    pe = torch.cat(ctx.pe)
    got, _ = w.forward_refined(None, s2w, custome_target_theta_embed=theta, custome_target_pose_embed=pe, **BASE)
    _, s1 = w.animate(theta, pe, **BASE)
    _u8_match(got, [s2w.forward(s1[i:i + 1])[2][0] for i in range(N)], "image-free")
    assert len(w._pipelines) <= w.PIPELINES
    # errors, refused before anything is queued
    with pytest.raises(ValueError, match="device"):
        w.forward_refined(ctx.drv[0], SimpleNamespace(model_two=SimpleNamespace(device=torch.device("cuda", 7), precision="exact")))
    with pytest.raises(TypeError):
        w.forward_refined(ctx.drv[0], s2w, smooth_pose=True)
    fresh = _wrapper(ctx)
    with pytest.raises(RuntimeError, match="source"):
        fresh.forward_refined(ctx.drv[0], s2w)


# ---- launch coverage --------------------------------------------------------------------------------------------------------
def test_refined_frame_launches_fall_in_tested_classes(s2_ckpt):
    """forward_refined live at 256^2 -> 512^2, exact and fast stage 2: every model launch is an entry of the launch tables,
    every boundary launch has a listed pattern, and the two handoff kernels run at shapes the kernel tests above check"""
    from emoportraits_b200 import lib as L

    ctx = _context(256)
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    s2s = [_s2_wrapper(s2_ckpt), _s2_wrapper(s2_ckpt, precision="fast")]
    lib = L.load()
    ops_table = {MOL.key(r) for r in MOL.load()}
    conv_table = {MCL.key(r) for r in MCL.load()}
    boundary_ops = {r["op"] for r in MOL.BOUNDARY}
    listed = {MOL.pattern(r) for r in MOL.BOUNDARY}
    seen = {"op": [], "conv": [], "boundary": [], "handoff": []}
    launch = L.call

    def call(name, *args):
        if name == "emo_conv_igemm":
            seen["conv"].append(MCL.launch_record(L, lib, args[0]._obj))
        elif name in ("emo_s2_prepare", "emo_s2_finish"):
            seen["handoff"].append((name, args))
        elif name[4:] in boundary_ops:
            seen["boundary"].append(MOL.launch_record(name, args))
        elif name not in MOL.NOT_RECORDED:
            seen["op"].append(MOL.launch_record(name, args))
        return launch(name, *args)

    pils = [FR.pil(256, 50 + i, "smooth") for i in range(3)]
    mp = pytest.MonkeyPatch()
    mp.setattr(L, "call", call)
    try:
        for s2w in s2s:
            w.forward_refined(pils, s2w, **BASE)
        torch.cuda.synchronize()
    finally:
        mp.undo()
    print(f"\n[refined frame launches] {len(seen['op'])} op, {len(seen['conv'])} conv, {len(seen['boundary'])} boundary, "
          f"{len(seen['handoff'])} handoff")
    assert seen["op"] and seen["conv"] and seen["boundary"] and seen["handoff"]
    assert not [r for r in seen["op"] if MOL.key(r) not in ops_table]
    assert not [r for r in seen["conv"] if MCL.key(r) not in conv_table]
    assert not [r for r in seen["boundary"] if MOL.pattern(r) not in listed]
    tested_prepare = {(h, w_, S) for _, h, w_, S in KERNEL_SHAPES}
    for name, args in seen["handoff"]:
        if name == "emo_s2_prepare":
            assert args[1] in (1, 2) and tuple(args[2:5]) in tested_prepare, args[:5]
        else:
            assert args[2] in (1, 2) and (args[3], args[4]) in {(512, 512), (1024, 1024), (517, 517)}, args[2:5]


def _batch1_1024_records(precision):
    """the stage-2 launches of a refined frame @1024^2 (Stage2Model.forward at batch 1 without its resize and stem_pack,
    tests/test_refine_stream_cpu.py), recorded in EMO_DRY_RUN mode: (conv records, op records) with their configuration"""
    from emoportraits_b200 import lib as L

    cfg = f"s2-1024-b1-{precision}"
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(L, "DRY_RUN", True)
        convs = MCL.record(cfg)
        op_recs = [r for r in MOL.record(cfg) if r["op"] not in ("resize_bilinear", "stem_pack")]
    return [dict(r, configs=[cfg]) for r in convs], [dict(r, configs=[cfg]) for r in op_recs]


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_batch1_1024_launches_replayed_against_float64(precision, monkeypatch):
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    convs, op_recs = _batch1_1024_records(precision)
    assert convs and op_recs
    conv_table = {MCL.key(r) for r in MCL.load()}
    ops_table = {MOL.key(r) for r in MOL.load()}
    new_convs = list({MCL.key(r): r for r in convs if MCL.key(r) not in conv_table}.values())
    new_ops = list({MOL.key(r): r for r in op_recs if MOL.key(r) not in ops_table}.values())
    print(f"\n[stage 2 batch 1 @1024^2 {precision}] {len(convs)} conv launches ({len(new_convs)} distinct not in the table), "
          f"{len(op_recs)} op launches ({len(new_ops)} distinct not in the table)")
    assert all(r["rc"] == 0 for r in convs), [r["err"] for r in convs if r["rc"]]
    monkeypatch.setattr(TMC, "ROWS", list(TMC.ROWS) + new_convs)
    monkeypatch.setattr(TMO, "ROWS", list(TMO.ROWS) + [("model", r) for r in new_ops])
    for k in range(len(new_convs)):
        TMC.test_model_conv_launch_against_float64((L, ops), len(TMC.ROWS) - len(new_convs) + k)
    for k in range(len(new_ops)):
        TMO.test_model_op_launch_against_float64((L, ops), len(TMO.ROWS) - len(new_ops) + k)
