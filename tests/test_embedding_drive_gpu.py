"""Driving captured frames from pose and expression embeddings on the GPU: DriverPipeline with the caller's pose (theta_embed),
expression embedding (pose_embed), both, both without a driver image, and encoding frames; InferenceWrapper.encode / animate
and forward with custome_target_theta_embed / custome_target_pose_embed.

Against the eager path (Model.driver_pass given the same tensors), with the in-flight rule of DESIGN.md section 2.4: every
frame of a sequence bit-identical but at most one, and that one within 5e-4.  Against the reference: the fixtures of
tests/golden/va256_options.pt within IMG_TOL.  Launch coverage: every launch encode, animate and the custom-embedding forward
issue is an entry of the tested model launch tables, or a wrapper-boundary launch of a listed pattern
(tests/test_model_op_launches_gpu.py)."""
import gc
import pathlib
from types import SimpleNamespace

import pytest
import torch

import model_conv_launches as MCL
import model_op_launches as MOL
from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
IMG_TOL = 1e-3          # tests/test_forward_options_gpu.py: max-abs per pixel against the reference's fixtures
N = 5
BASE = dict(mix=True, mix_old=False)     # the video loop's options (video.drive_image_with_video)
INPUTS = {"theta": dict(theta_embed=True), "pose": dict(pose_embed=True), "both": dict(theta_embed=True, pose_embed=True),
          "image_free": dict(image=False, theta_embed=True, pose_embed=True), "encode": dict(encode=True)}
OPTIONS = {"mix": dict(mix=True), "no_mix": dict(mix=False), "target_theta_false": dict(mix=True, target_theta=False),
           "mix_old": dict(mix=True, mix_old=True)}


@pytest.fixture(autouse=True)
def _release():
    """after each test, collect its wrappers and captured graphs here, with no capture in progress: a graph that waits for
    the cyclic garbage collector may otherwise be destroyed in the middle of a later test's capture (see
    Model._make_driver_graph), and its ~3.6 GB per pipeline would stay reserved"""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _match(got, want, what=""):
    errs = [(g.float().cpu() - w.float().cpu()).abs().max().item() for g, w in zip(got, want)]
    assert len(errs) == len(want) and max(errs) < 5e-4 and sum(e == 0.0 for e in errs) >= len(errs) - 1, (what, errs)


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
    # realistic inputs: frame i takes the regressed pose of frame i + 1 and the embedding of frame i + 2
    enc = [model.driver_pass(st["A"], d, mix=True, encode_only=True)[3] for d in drv]
    srt = [enc[(i + 1) % N].srt.clone() for i in range(N)]
    pe = [enc[(i + 2) % N].target_pose_embed.clone() for i in range(N)]
    return SimpleNamespace(size=size, cfg=cfg, sd=sd, hsd=hsd, model=model, src=src, st=st, drv=drv, srt=srt, pe=pe)


@pytest.fixture(scope="module")
def ctx():
    return _context(256)


def _wrapper(ctx, **kw):
    from emoportraits_b200.infer import InferenceWrapper

    return InferenceWrapper("embed", args_path=GOLD / f"args_{ctx.size}.txt", state_dict=ctx.sd, head_pose_state_dict=ctx.hsd,
                            print_params=False, **kw)


def _pils(ctx, n=N):
    return [FR.pil(ctx.size, 50 + i, "smooth") for i in range(n)]


def _frame_args(ctx, i, flags):
    return dict(drv=ctx.drv[i] if flags.get("image", True) else None,
                theta_embed=ctx.srt[i] if flags.get("theta_embed") else None,
                pose_embed=ctx.pe[i] if flags.get("pose_embed") else None)


# ---- Model / DriverPipeline -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", list(OPTIONS))
@pytest.mark.parametrize("inp", list(INPUTS))
def test_captured_frame_matches_eager(ctx, inp, opt):
    """every input set under every pose option: five captured frames, two in flight, against the eager pass given the same
    tensors (an encoding frame: its pose and embedding against the eager encoding and the whole eager frame's)"""
    from emoportraits_b200.infer import DriverPipeline

    kw, flags = OPTIONS[opt], INPUTS[inp]
    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=2, **kw, **flags)
    encode = flags.get("encode", False)
    s = ctx.size
    outs = [torch.empty((1, 3, s, s), device="cuda") for _ in range(N)]
    srt, pe = torch.empty((N, 9), device="cuda"), torch.empty((N, ctx.cfg.expr_channels), device="cuda")
    for i in range(N):
        a = _frame_args(ctx, i, flags)
        sl = pipe.submit(a.pop("drv"), dev_out=None if encode else outs[i], **a).slot
        if encode:
            with torch.cuda.stream(sl.stream):
                srt[i:i + 1].copy_(sl.run.static_state.srt)
                pe[i:i + 1].copy_(sl.run.static_state.target_pose_embed)
    pipe.drain()
    torch.cuda.synchronize()
    want = []
    for i in range(N):
        a = _frame_args(ctx, i, flags)
        want.append(ctx.model.driver_pass(ctx.st["A"], a["drv"], custom_srt=a["theta_embed"], custom_pose_embed=a["pose_embed"],
                                          encode_only=encode, **kw))
    if encode:
        _match([srt[i:i + 1] for i in range(N)], [w[3].srt for w in want], "srt")
        _match([pe[i:i + 1] for i in range(N)], [w[3].target_pose_embed for w in want], "pose_embed")
        full = [ctx.model.driver_pass(ctx.st["A"], d, **kw)[3] for d in ctx.drv]
        assert all(torch.equal(w[3].srt, f.srt) and torch.equal(w[3].target_pose_embed, f.target_pose_embed)
                   for w, f in zip(want, full))
    else:
        _match(outs, [w[0] for w in want], (inp, opt))
        so = pipe.slots[(N - 1) % 2].run.static_state
        last = want[-1][3]
        assert torch.equal(so.srt, last.srt) and torch.equal(so.target_pose_embed, last.target_pose_embed)


def test_image_free_interleaved_identities(ctx):
    """image-free frames of A and B interleaved, four in flight (st= per frame): each matches its own identity's eager frame"""
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=4, image=False, theta_embed=True, pose_embed=True, **BASE)
    order = "ABBABAAB"
    outs = [torch.empty((1, 3, ctx.size, ctx.size), device="cuda") for _ in order]
    for k, who in enumerate(order):
        pipe.submit(None, dev_out=outs[k], st=ctx.st[who], theta_embed=ctx.srt[k % N], pose_embed=ctx.pe[k % N])
    pipe.drain()
    torch.cuda.synchronize()
    want = [ctx.model.driver_pass(ctx.st[who], None, custom_srt=ctx.srt[k % N], custom_pose_embed=ctx.pe[k % N], **BASE)[0]
            for k, who in enumerate(order)]
    _match(outs, want)
    assert (want[0] - want[1]).abs().max().item() > 1e-2     # the identities differ visibly


# ---- InferenceWrapper -------------------------------------------------------------------------------------------------
def _split(img):
    return [img[i:i + 1] for i in range(img.shape[0])]


def _roundtrip(ctx, w, pils, kw):
    """animate(*encode(frames)) against forward(None, frames); the attributes each sets"""
    _, want = w.forward(None, pils, crop=False, **kw)
    want_srt = torch.cat(w.pred_target_srt, 1)
    want_theta = w.pred_target_theta
    theta, pe = w.encode(pils, **kw)
    assert all(t.shape == (len(pils), 3) for t in theta) and pe.shape == (len(pils), ctx.cfg.expr_channels)
    assert torch.equal(torch.cat([t[-1:] for t in theta], 1), want_srt)
    pil, got = w.animate(theta, pe, **kw)
    assert len(pil) == len(pils) and got.shape == want.shape
    _match(_split(got), _split(want), kw)
    assert torch.equal(torch.cat(w.pred_target_srt, 1), want_srt) and torch.equal(w.target_pose_embed, pe[-1:])
    assert torch.equal(w.pred_target_theta, want_theta)
    return theta, pe


def test_animate_encode_roundtrip(ctx):
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    pils = _pils(ctx)
    for kw in (BASE, dict(), dict(mix=True, mix_old=True), dict(mix=True, target_theta=False)):
        theta, pe = _roundtrip(ctx, w, pils, kw)
    # a tensor batch encodes as its frames one at a time do
    theta_t, pe_t = w.encode(torch.cat(ctx.drv), **BASE)
    one = [w.encode(d, **BASE) for d in ctx.drv]
    _match(_split(pe_t), [p for _, p in one])
    _match(_split(torch.cat(theta_t, 1)), [torch.cat(t, 1) for t, _ in one])
    # the embedding depends on the mixing: encoded with mix=False it differs
    _, pe_nomix = w.encode(pils, mix=False)
    assert (pe_nomix - pe).abs().max().item() > 1e-4


def test_forward_custom_embeddings_match_eager(ctx):
    """forward(None, frames, custome_target_pose_embed=e) / custome_target_theta_embed: the captured frames against one
    eager call per frame; pred_target_srt stays the regressed pose"""
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    pils = _pils(ctx)
    e = ctx.pe[0]
    theta = (ctx.srt[0][:, :3].cpu(), ctx.srt[0][:, 3:6].cpu(), ctx.srt[0][:, 6:9].cpu())
    for kw in (dict(custome_target_pose_embed=e), dict(custome_target_theta_embed=theta),
               dict(custome_target_pose_embed=e.cpu().reshape(-1), custome_target_theta_embed=theta)):
        custom = dict(custom_srt=torch.cat(theta, 1) if "custome_target_theta_embed" in kw else None,
                      custom_pose_embed=kw.get("custome_target_pose_embed"))
        eager = [w.model.driver_pass(w.identity, w._prep(p), **custom, **BASE) for p in pils]
        _, got = w.forward(None, pils, crop=False, **kw, **BASE)
        _match(_split(got), [x[0] for x in eager], list(kw))
        assert torch.equal(torch.cat(w.pred_target_srt, 1), eager[-1][3].srt)          # regressed, not the supplied pose
        _, one = w.forward(None, pils[1], crop=False, **kw, **BASE)
        _match([one], [eager[1][0]], list(kw))
        assert torch.equal(w.target_pose_embed, eager[1][3].target_pose_embed)
        assert torch.equal(w.pred_target_theta, eager[1][3].pred_target_theta)


def test_fast_precision_animate(ctx):
    w = _wrapper(ctx, precision="fast")
    w.forward(ctx.src["B"], None, crop=False)
    theta = tuple(torch.cat([s[:, k:k + 3] for s in ctx.srt]) for k in (0, 3, 6))
    pe = torch.cat(ctx.pe)
    _, got = w.animate(theta, pe, **BASE)
    want = [w.model.driver_pass(w.identity, None, custom_srt=ctx.srt[i], custom_pose_embed=ctx.pe[i], **BASE)[0] for i in range(N)]
    _match(_split(got), want)
    assert w.model.decoder_nw.planes != ctx.model.decoder_nw.planes


# ---- against the reference's fixtures ---------------------------------------------------------------------------------
def test_reference_fixtures(ctx):
    from emoportraits_b200.config import shipped_config
    from oracle.make_golden import option_inputs

    full = torch.load(GOLD / "va256_options.pt", weights_only=False)
    gold, X = full["cases"], option_inputs(256, shipped_config(256))

    def err(img, case):
        vals, stride = case["img"]
        return (img.detach().float().cpu().reshape(-1)[::stride] - vals).abs().max().item()

    w = _wrapper(ctx)
    src = FR.pil(256, full["src_seed"], full["kind"])
    drv = FR.pil(256, full["drv_seeds"][0], full["kind"])
    base = dict(crop=False, mix=True, mix_old=False)
    _, img = w.forward(src, drv, custome_target_theta_embed=X["theta_embed"], **base)
    assert err(img, gold["custome_target_theta_embed"]) < IMG_TOL
    _, img = w.forward(None, drv, custome_target_pose_embed=X["pose_embed"], **base)
    case = gold["custome_target_pose_embed"]
    assert err(img, case) < IMG_TOL
    regressed = w.pred_target_srt
    _, img = w.animate(regressed, case["target_pose_embed"].reshape(1, -1), mix=True, mix_old=False)
    assert err(img, case) < IMG_TOL
    assert (w.pred_target_theta[:, :3].cpu() - case["pred_target_theta"][:, :3]).abs().max().item() < 1e-5


# ---- launch coverage ------------------------------------------------------------------------------------------------------
def test_launches_fall_in_tested_classes():
    """encode, animate and the custom-embedding forward run live at 256^2: every model launch is an entry of the tested
    launch tables (tests/model_op_launches.json, tests/model_conv_launches.json), every boundary launch has a listed pattern"""
    from emoportraits_b200 import lib as L

    ctx = _context(256)
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    lib = L.load()
    ops_table = {MOL.key(r) for r in MOL.load()}
    conv_table = {MCL.key(r) for r in MCL.load()}
    boundary_ops = {r["op"] for r in MOL.BOUNDARY}
    listed = {MOL.pattern(r) for r in MOL.BOUNDARY}
    seen = {"op": [], "conv": [], "boundary": []}
    launch = L.call

    def call(name, *args):
        if name == "emo_conv_igemm":
            seen["conv"].append(MCL.launch_record(L, lib, args[0]._obj))
        elif name[4:] in boundary_ops:
            seen["boundary"].append(MOL.launch_record(name, args))
        elif name not in MOL.NOT_RECORDED:
            seen["op"].append(MOL.launch_record(name, args))
        return launch(name, *args)

    pils = _pils(ctx, 3)
    mp = pytest.MonkeyPatch()
    mp.setattr(L, "call", call)
    try:
        theta, pe = w.encode(pils, **BASE)
        w.animate(theta, pe, **BASE)
        w.forward(None, pils, crop=False, custome_target_pose_embed=pe[0], **BASE)
        w.forward(None, pils[0], crop=False, custome_target_theta_embed=tuple(t[:1] for t in theta), **BASE)
        torch.cuda.synchronize()
    finally:
        mp.undo()
    print(f"\n[embedding drive launches] {len(seen['op'])} op, {len(seen['conv'])} conv, {len(seen['boundary'])} boundary")
    assert seen["op"] and seen["conv"] and seen["boundary"]
    assert not [r for r in seen["op"] if MOL.key(r) not in ops_table]
    assert not [r for r in seen["conv"] if MCL.key(r) not in conv_table]
    assert not [r for r in seen["boundary"] if MOL.pattern(r) not in listed]


# ---- the flagship size ----------------------------------------------------------------------------------------------------
def test_flagship_size():
    """@512^2: animate(*encode(frames)) against forward(None, frames), and the custom-embedding forward against eager frames"""
    ctx = _context(512)
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    pils = _pils(ctx)
    _roundtrip(ctx, w, pils, BASE)
    _, got = w.forward(None, pils, crop=False, custome_target_pose_embed=ctx.pe[0], **BASE)
    want = [w.model.driver_pass(w.identity, w._prep(p), custom_pose_embed=ctx.pe[0], **BASE)[0] for p in pils]
    _match(_split(got), want)
