"""Smoothed frames in flight on the GPU: DriverPipeline(smooth=True) with PoseTracks and InferenceWrapper.forward(list,
smooth_pose=True).

  * Pipeline: depth 4, 10 frames (not a multiple of the depth) on each of three tracks at momenta 0.1 / 0.5 / 0.9,
    interleaved frame by frame, for mix on and off, mix_old and target_theta=False: every frame's pred_target_theta and each
    track's final state are torch.equal to the eager driver_pass(smooth_state=...) recurrence (the pose step is one thread's
    fp32 arithmetic on the bits the unsmoothed launch wrote), and every image is torch.equal to the sequential captured
    smoothing frames (the wrapper's single-frame path) and meets the in-flight rule against eager.
  * Four tracks on two identities, interleaved frame by frame: each equals its own sequential recurrence.
  * Wrapper: a forward(list) call, single-frame calls, another list and a reset_tracking list: one continuous recurrence, with
    self.theta and pred_target_theta those of the eager recurrence after every call.
  * The reference's fixture (tests/golden/va256_options.pt): its drivers through one forward(list, smooth_pose=True,
    reset_tracking=True) call against the smooth_pose_i records, at the bars of tests/test_forward_options_gpu.py.
  * Refine: a smoothing pipeline with refine= equals stage 2 applied to its own smoothed stage-1 frames.
  * Launch coverage: the model launches of smoothed frames in flight are entries of the tested launch tables, and the pose
    step falls in the "pose_theta theta_in nomix smooth" class of tests/op_cases.py."""
import gc
import pathlib
from types import SimpleNamespace

import pytest
import torch

import model_conv_launches as MCL
import model_op_launches as MOL
import op_cases as OC
from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
N = 10
DEPTH = 4
MOMENTA = (0.1, 0.5, 0.9)
BASE = dict(mix=True, mix_old=False)
OPTIONS = [dict(mix=True), dict(mix=False), dict(mix=True, mix_old=True), dict(mix=True, target_theta=False)]
IMG_TOL = 1e-3      # tests/test_forward_options_gpu.py
THETA_TOL = 1e-5


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _assert_match(got, want, what=""):
    """the in-flight rule of tests/test_identity_switch_gpu.py"""
    errs = [(g.float().cpu() - w.float().cpu()).abs().max().item() for g, w in zip(got, want)]
    assert len(errs) == len(want) and max(errs) < 5e-4 and sum(e == 0.0 for e in errs) >= len(errs) - 1, (what, errs)


@pytest.fixture(scope="module")
def ctx():
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    size = 256
    cfg = shipped_config(size)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    model = Model(cfg, sd, hsd, "cuda")
    src = {k: FR.frame(size, s, "smooth").cuda() for k, s in {"A": 41, "B": 61}.items()}
    st = {k: model.source_pass(x) for k, x in src.items()}
    drv = [FR.frame(size, 50 + i, "smooth").cuda() for i in range(N)]
    return SimpleNamespace(size=size, cfg=cfg, sd=sd, hsd=hsd, model=model, src=src, st=st, drv=drv)


def _eager(model, st, frames, m, **opt):
    """the eager smoothing recurrence: (images, pred_target_theta per frame, final state)"""
    state = torch.zeros((3, 4), device="cuda")
    imgs, thetas = [], []
    for i, d in enumerate(frames):
        img, _, _, so = model.driver_pass(st, d, smooth_state=state, smooth_momentum=m, smooth_init=(i == 0), **opt)
        imgs.append(img.clone())
        thetas.append(so.pred_target_theta.clone())
    return imgs, thetas, state


def _sequential(model, st, frames, m, **opt):
    """the sequential captured smoothing frames (the wrapper's single-frame path): the first frame seeds the state eagerly,
    the others replay one captured graph that smooths into it"""
    state = torch.zeros((3, 4), device="cuda")
    imgs = [model.driver_pass(st, frames[0], smooth_state=state, smooth_momentum=m, smooth_init=True, **opt)[0].clone()]
    run = model.make_driver_graph(st, smooth_state=state, smooth_momentum=m, **opt)
    imgs += [run(d).clone() for d in frames[1:]]
    torch.cuda.synchronize()
    del run
    return imgs, state


def _submit_all(pipe, seq):
    """seq: (frame, track, st or None) per frame; returns per frame (image, pred_target_theta) copied on the frame's stream"""
    s = pipe.model.cfg.image_size
    out = []
    for d, tr, st in seq:
        o = (torch.empty((1, 3, s, s), device="cuda"), torch.empty((1, 4, 4), device="cuda"))
        t = pipe.submit(d, dev_out=o[0], track=tr, st=st)
        with torch.cuda.stream(t.slot.stream):
            o[1].copy_(t.slot.run.static_state.pred_target_theta)
        out.append(o)
    pipe.drain()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("opt", OPTIONS, ids=["mix", "no_mix", "mix_old", "target_theta_false"])
def test_tracks_match_the_sequential_recurrence(ctx, opt):
    from emoportraits_b200.infer import DriverPipeline

    st = ctx.st["A"]
    pipe = DriverPipeline(ctx.model, st, depth=DEPTH, smooth=True, **opt)
    tracks = [pipe.track(momentum=m) for m in MOMENTA]
    got = _submit_all(pipe, [(ctx.drv[i], tracks[k], None) for i in range(N) for k in range(len(MOMENTA))])
    for k, m in enumerate(MOMENTA):
        mine = got[k::len(MOMENTA)]
        imgs, thetas, state = _eager(ctx.model, st, ctx.drv, m, **opt)
        for i in range(N):
            assert torch.equal(mine[i][1], thetas[i]), (opt, m, i)
        assert torch.equal(tracks[k].state, state), (opt, m)
        seq_imgs, seq_state = _sequential(ctx.model, st, ctx.drv, m, **opt)
        assert torch.equal(seq_state, state)
        for i in range(N):
            assert torch.equal(mine[i][0], seq_imgs[i]), (opt, m, i)
        _assert_match([g[0] for g in mine], imgs, (opt, m))
    # the momenta make different recurrences
    assert not torch.equal(tracks[0].state, tracks[2].state)


def test_four_tracks_two_identities(ctx):
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=DEPTH, smooth=True, **BASE)
    who = ["A", "B", "A", "B"]
    tracks = [pipe.track(momentum=m) for m in (0.5, 0.5, 0.9, 0.3)]
    n = 6
    # track k reads the frames from k on: the four recurrences differ
    seq = [(ctx.drv[(i + k) % N], tracks[k], ctx.st[who[k]]) for i in range(n) for k in range(4)]
    got = _submit_all(pipe, seq)
    for k in range(4):
        mine = got[k::4]
        imgs, thetas, state = _eager(ctx.model, ctx.st[who[k]], [ctx.drv[(i + k) % N] for i in range(n)], tracks[k].momentum, **BASE)
        assert all(torch.equal(mine[i][1], thetas[i]) for i in range(n)), k
        assert torch.equal(tracks[k].state, state), k
        _assert_match([g[0] for g in mine], imgs, k)
    # a reset seeds the track again: its next frames are a new recurrence
    tracks[1].reset()
    got = _submit_all(pipe, [(ctx.drv[i], tracks[1], ctx.st["B"]) for i in range(5)])
    imgs, thetas, state = _eager(ctx.model, ctx.st["B"], ctx.drv[:5], 0.5, **BASE)
    assert all(torch.equal(g[1], t) for g, t in zip(got, thetas)) and torch.equal(tracks[1].state, state)
    _assert_match([g[0] for g in got], imgs)


def _wrapper(ctx, **kw):
    from emoportraits_b200.infer import InferenceWrapper

    return InferenceWrapper("smooth", args_path=GOLD / f"args_{ctx.size}.txt", state_dict=ctx.sd, head_pose_state_dict=ctx.hsd,
                            print_params=False, **kw)


def test_wrapper_one_continuous_recurrence(ctx):
    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    pils = [FR.pil(ctx.size, 50 + i, "smooth") for i in range(N)]
    frames = [w._prep(p) for p in pils]
    m = w.pose_momentum
    state = torch.zeros((3, 4), device="cuda")
    eager = []

    def step(i, init):
        img, _, _, so = w.model.driver_pass(w.identity, frames[i], smooth_state=state, smooth_momentum=m, smooth_init=init, **BASE)
        eager.append(img.clone())
        return so.pred_target_theta.clone()

    def check(img, first, theta):
        assert torch.equal(w.theta, state) and torch.equal(w.pred_target_theta, theta)
        _assert_match(list(img.split(1)), eager[first:])

    _, img = w.forward(None, pils[:5], crop=False, smooth_pose=True, reset_tracking=True, **BASE)
    theta = [step(i, i == 0) for i in range(5)][-1]
    check(img, 0, theta)
    for i in (5, 6):
        _, img = w.forward(None, pils[i], crop=False, smooth_pose=True, **BASE)     # one captured graph, the same state
        theta = step(i, False)
        check(img, i, theta)
    _, img = w.forward(None, torch.cat(frames[7:]), crop=False, smooth_pose=True, **BASE)   # a batch: in flight again
    theta = [step(i, False) for i in range(7, N)][-1]
    check(img, 7, theta)
    eager.clear()
    state.zero_()
    _, img = w.forward(None, pils[2:6], crop=False, smooth_pose=True, reset_tracking=True, **BASE)
    theta = [step(i, i == 2) for i in range(2, 6)][-1]
    check(img, 0, theta)


def test_reference_fixture(ctx):
    full = torch.load(GOLD / "va256_options.pt", weights_only=False)
    gold = full["cases"]
    w = _wrapper(ctx)
    src = FR.pil(256, full["src_seed"], full["kind"])
    drv = [FR.pil(256, s, full["kind"]) for s in full["drv_seeds"]]
    assert len(drv) > 1
    w.forward(src, None, crop=False, **BASE)
    _, img = w.forward(None, drv, crop=False, smooth_pose=True, reset_tracking=True, **BASE)
    for i in range(len(drv)):
        vals, stride = gold[f"smooth_pose_{i}"]["img"]
        err = (img[i].detach().float().cpu().reshape(-1)[::stride] - vals).abs().max().item()
        assert err < IMG_TOL, (i, err)
    last = gold[f"smooth_pose_{len(drv) - 1}"]["pred_target_theta"]
    assert (w.pred_target_theta[:, :3].cpu() - last[:, :3]).abs().max().item() < THETA_TOL
    assert (w.theta.cpu() - last[0, :3]).abs().max().item() < THETA_TOL


def test_refined_smoothed_frames(ctx):
    from emoportraits_b200 import ops
    from emoportraits_b200.infer import DriverPipeline
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2

    cfg2 = Stage2Config(output_size=512)
    s2 = Stage2Model(cfg2, synthetic_state_dict_s2(cfg2, 0), "cuda", precision="exact")
    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=2, smooth=True, refine=s2, **BASE)
    tr = pipe.track(momentum=0.5)
    got = []
    for d in ctx.drv[:5]:
        o = (torch.empty((1, 3, 512, 512), device="cuda"), torch.empty((1, 512, 512, 3), dtype=torch.uint8, device="cuda"),
             torch.empty((1, 3, 256, 256), device="cuda"))
        t = pipe.submit(d, dev_out=o[0], u8_out=o[1], track=tr)
        with torch.cuda.stream(t.slot.stream):
            o[2].copy_(t.slot.run.static_stage1)
        got.append(o)
    pipe.drain()
    torch.cuda.synchronize()
    imgs, _, state = _eager(ctx.model, ctx.st["A"], ctx.drv[:5], 0.5, **BASE)
    assert torch.equal(tr.state, state)
    _assert_match([g[2] for g in got], imgs)
    for k, (ref_img, u8, s1) in enumerate(got):
        ffhq = s2.forward(s1)[2]
        assert torch.equal(ref_img, ffhq), k
        assert torch.equal(u8, ops.image_to_u8(ffhq)), k


def test_launches_fall_in_tested_classes(ctx):
    """smoothed frames in flight at 256^2 through forward(list) and a DriverPipeline with two tracks: every model launch is an
    entry of the tested launch tables, every boundary launch has a listed pattern, and the pose step is a launch of the
    smoothing class its cases in tests/op_cases.py check against float64"""
    from emoportraits_b200 import lib as L
    from emoportraits_b200.infer import DriverPipeline

    w = _wrapper(ctx)
    w.forward(ctx.src["A"], None, crop=False)
    pils = [FR.pil(ctx.size, 50 + i, "smooth") for i in range(6)]
    lib = L.load()
    ops_table = {MOL.key(r) for r in MOL.load()}
    conv_table = {MCL.key(r) for r in MCL.load()}
    boundary_ops = {r["op"] for r in MOL.BOUNDARY}
    listed = {MOL.pattern(r) for r in MOL.BOUNDARY}
    seen = {"op": [], "conv": [], "boundary": [], "step": []}
    launch = L.call

    def call(name, *args):
        if name == "emo_conv_igemm":
            seen["conv"].append(MCL.launch_record(L, lib, args[0]._obj))
        elif name[4:] in boundary_ops:
            seen["boundary"].append(MOL.launch_record(name, args))
        elif name == "emo_pose_theta" and args[0]._obj.smooth_state:
            seen["step"].append(MOL.launch_record(name, args))
        elif name not in MOL.NOT_RECORDED:
            seen["op"].append(MOL.launch_record(name, args))
        return launch(name, *args)

    mp = pytest.MonkeyPatch()
    mp.setattr(L, "call", call)
    try:
        w.forward(None, pils, crop=False, smooth_pose=True, reset_tracking=True, **BASE)
        pipe = DriverPipeline(w.model, w.identity, depth=DEPTH, smooth=True, **BASE)
        tracks = [pipe.track(momentum=0.9), pipe.track(momentum=0.3)]
        for i in range(6):
            pipe.submit(w._prep(pils[i]), track=tracks[i % 2])
        pipe.drain()
        torch.cuda.synchronize()
    finally:
        mp.undo()
    print(f"\n[smoothed in flight launches] {len(seen['op'])} op, {len(seen['conv'])} conv, {len(seen['boundary'])} boundary, "
          f"{len(seen['step'])} pose steps")
    assert seen["op"] and seen["conv"] and seen["boundary"] and len(seen["step"]) >= 12
    assert not [r for r in seen["op"] if MOL.key(r) not in ops_table]
    assert not [r for r in seen["conv"] if MCL.key(r) not in conv_table]
    assert not [r for r in seen["boundary"] if MOL.pattern(r) not in listed]
    assert {r["cls"] for r in seen["step"]} == {"pose_theta theta_in nomix smooth"}
    assert "pose_theta theta_in nomix smooth" in {c.want for c in OC.CASES}
    # the momenta, seeding and carrying, are among those the pose cases check
    feats = {f for r in seen["step"] for f in r["features"]}
    assert {"smooth init", "smooth carried", "momentum 0.5 init", "momentum 0.9 carried", "momentum 0.3 carried"} <= feats
    assert {0.5, 0.9, 0.3} <= set(OC.POSE_MOMENTA)
