"""Identity switching on the GPU: captured driver graphs that load a new source identity into buffers of their own instead of
being re-captured (Model.make_driver_graph, replay.load), several identities in flight in one DriverPipeline
(submit(..., st=)), and InferenceWrapper keeping its graphs across source passes (forward(new_source, driver), the
`identity` handle, smooth_pose).

The reference for every frame is the plain eager Model.driver_pass on the frame's own source state.  The rule is the one of
tests/test_model_gpu.py::test_frames_in_flight_match_sequential: every frame of a sequence bit-identical but at most one, and
that one within 5e-4 (a stale or half-copied identity, or scratch shared between passes in flight, shows up as 1e-2+).  The
identities do differ by more than 1e-2, so a frame of the wrong identity cannot pass."""
import pathlib
from types import SimpleNamespace

import pytest
import torch

from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
SRC_SEEDS = {"A": 41, "B": 61, "C": 71}
BASE = dict(mix=True, mix_old=False)     # the wrapper's options in the video loop (video.drive_image_with_video)


def _assert_match(got, want, what=""):
    errs = [(g.float().cpu() - w.float().cpu()).abs().max().item() for g, w in zip(got, want)]
    assert len(errs) == len(want) and max(errs) < 5e-4 and sum(e == 0.0 for e in errs) >= len(errs) - 1, (what, errs)


@pytest.fixture(scope="module", params=[256, 512])
def ctx(request):
    size = request.param
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    cfg = shipped_config(size)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    model = Model(cfg, sd, hsd, "cuda")
    src = {k: FR.frame(size, s, "smooth").cuda() for k, s in SRC_SEEDS.items()}
    states = {k: model.source_pass(x) for k, x in src.items()}
    drv = [FR.frame(size, 50 + i, "smooth").cuda() for i in range(6)]
    cache = {}

    def eager(who, i, **kw):
        """the eager image of identity `who` driven by frame i"""
        key = (who, i, tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = model.driver_pass(states[who], drv[i], **kw)[0].clone()
        return cache[key]

    a, b = eager("A", 0, mix=True), eager("B", 0, mix=True)
    assert (a - b).abs().max().item() > 1e-2   # the identities differ visibly
    return SimpleNamespace(size=size, cfg=cfg, sd=sd, hsd=hsd, model=model, src=src, st=states, drv=drv, eager=eager)


@pytest.fixture
def captures(monkeypatch):
    """counts Model._make_driver_graph calls (one per captured graph)"""
    from emoportraits_b200.infer import Model

    n = [0]
    orig = Model._make_driver_graph

    def counted(self, *a, **k):
        n[0] += 1
        return orig(self, *a, **k)

    monkeypatch.setattr(Model, "_make_driver_graph", counted)
    return n


def _run(pipe, ctx, seq, **kw):
    """submit (identity, frame index) pairs through `pipe`; returns the images after a drain"""
    outs = [torch.empty((1, 3, ctx.size, ctx.size), device="cuda") for _ in seq]
    for (who, i), o in zip(seq, outs):
        pipe.submit(ctx.drv[i], dev_out=o, st=ctx.st[who] if who else None)
    pipe.drain()
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("kw", [dict(mix=True), dict(mix=False), dict(mix=True, target_theta=False), dict(mix=True, mix_old=True)],
                         ids=["mix", "no_mix", "target_theta_false", "mix_old"])
def test_capture_once_switch(ctx, captures, kw):
    """a pipeline captured for A drives B and then A again: no capture after the constructor's, every frame its identity's"""
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=2, **kw)
    assert captures[0] == 2
    seq = [("B", 0), (None, 1), (None, 2), ("A", 3), (None, 4), ("B", 5), ("A", 0)]
    who = ["B", "B", "B", "A", "A", "B", "A"]
    got = _run(pipe, ctx, seq)
    _assert_match(got, [ctx.eager(w, i, **kw) for w, (_, i) in zip(who, seq)], kw)
    assert captures[0] == 2 and pipe.st is ctx.st["A"]


def test_interleaved_identities(ctx, captures):
    """four frames in flight, each of the next identity in A B C A B A C ...: every frame matches its own identity"""
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=4, mix=True)
    order = "ABCABACCBABC"
    seq = [(w, k % len(ctx.drv)) for k, w in enumerate(order)]
    got = _run(pipe, ctx, seq)
    _assert_match(got, [ctx.eager(w, i, mix=True) for w, i in seq])
    assert captures[0] == 4


def test_source_pass_during_flight(ctx):
    """A's frames in flight while B's source pass runs on the current stream (eager scratch set 0, apart from the slots'),
    then B's frames: both identities' frames and B's state match the undisturbed ones"""
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=4, mix=True)
    outs = [torch.empty((1, 3, ctx.size, ctx.size), device="cuda") for _ in range(10)]
    for k in range(6):
        pipe.submit(ctx.drv[k], dev_out=outs[k])
    st_b = ctx.model.source_pass(ctx.src["B"])          # no drain: A's frames are still running
    for k in range(4):
        pipe.submit(ctx.drv[k], dev_out=outs[6 + k], st=st_b)
    pipe.drain()
    torch.cuda.synchronize()
    _assert_match(outs, [ctx.eager("A", k, mix=True) for k in range(6)] + [ctx.eager("B", k, mix=True) for k in range(4)])
    assert torch.equal(st_b.target_latent_volume, ctx.st["B"].target_latent_volume)


def test_dropped_identity_stays_valid_until_loaded(ctx):
    """B's frames queued behind busy slots, then A's on every slot: the pipeline and the caller both let go of B before its
    copies ran; its memory is released, re-allocated and overwritten, and B's frames are still B's"""
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=4, mix=True)
    outs = [torch.empty((1, 3, ctx.size, ctx.size), device="cuda") for _ in range(12)]
    st_b = ctx.model.source_pass(ctx.src["B"])
    torch.cuda.synchronize()
    nbytes = sum(t.numel() for t in vars(st_b).values() if isinstance(t, torch.Tensor))
    for k in range(4):
        pipe.submit(ctx.drv[k], dev_out=outs[k])
    for k in range(4):
        pipe.submit(ctx.drv[k], dev_out=outs[4 + k], st=st_b)
    for k in range(4):
        pipe.submit(ctx.drv[k], dev_out=outs[8 + k], st=ctx.st["A"])
    del st_b
    torch.cuda.empty_cache()
    junk = torch.full((nbytes,), 1e3, device="cuda")
    pipe.drain()
    torch.cuda.synchronize()
    del junk
    want = [ctx.eager(w, k, mix=True) for w in "ABA" for k in range(4)]
    _assert_match(outs, want)


def test_broadcast_state_loads(ctx, monkeypatch):
    """a state rebuilt by dist.broadcast_source_state (here with a one-process stand-in for the collective) loads into a
    pipeline and drives B's frames"""
    from emoportraits_b200 import dist as D
    from emoportraits_b200.infer import DriverPipeline

    monkeypatch.setattr(D.dist, "get_rank", lambda group=None: 0)
    monkeypatch.setattr(D.dist, "broadcast", lambda t, src=0, group=None: None)
    st_b = D.broadcast_source_state(ctx.st["B"], ctx.cfg, "cuda", src=0)
    assert set(vars(st_b)) == {"target_latent_volume", "idt_embed", "pred_source_theta", "source_theta_dev"}
    pipe = DriverPipeline(ctx.model, ctx.st["A"], depth=2, mix=True)
    outs = [torch.empty((1, 3, ctx.size, ctx.size), device="cuda") for _ in range(4)]
    for k in range(4):
        pipe.submit(ctx.drv[k], dev_out=outs[k], st=st_b if k % 2 == 0 else ctx.st["A"])
    pipe.drain()
    torch.cuda.synchronize()
    _assert_match(outs, [ctx.eager("BA"[k % 2], k, mix=True) for k in range(4)])


# ---- InferenceWrapper -------------------------------------------------------------------------------------------------
def _wrapper(ctx, **kw):
    from emoportraits_b200.infer import InferenceWrapper

    return InferenceWrapper("identity", args_path=GOLD / f"args_{ctx.size}.txt", state_dict=ctx.sd, head_pose_state_dict=ctx.hsd,
                            print_params=False, **kw)


CACHED = ("idt_embed", "pred_source_theta", "pred_source_pose_embed", "source_latent_volume", "source_xy_warp_resize",
          "target_latent_volume_1", "target_latent_volume", "source_image", "source_image_crop", "source_img_mask", "source_img",
          "source_img_crop_m")


@pytest.mark.parametrize("prec", [dict(), dict(precision="fast"), dict(source_precision="fast")],
                         ids=["exact", "fast", "source_fast"])
def test_wrapper_photo_to_photo_captures_once(ctx, captures, prec):
    """forward(src_A, drv) then forward(src_B, drv): the second call captures nothing, and its image is a fresh wrapper's"""
    if prec and ctx.size != 512:
        pytest.skip("the precision settings run at the flagship size")
    w = _wrapper(ctx, **prec)
    d = ctx.drv[0]
    _, img_a = w.forward(ctx.src["A"], d, crop=False, **BASE)
    assert captures[0] == 4
    _, img_b = w.forward(ctx.src["B"], d, crop=False, **BASE)
    assert captures[0] == 4
    _, img_a2 = w.forward(ctx.src["A"], d, crop=False, **BASE)
    assert captures[0] == 4
    fresh = _wrapper(ctx, **prec)
    _, want_b = fresh.forward(ctx.src["B"], d, crop=False, **BASE)
    _assert_match([img_b, img_a2], [want_b, img_a])
    _assert_match([img_b], [fresh.model.driver_pass(fresh.identity, d, **BASE)[0]])
    assert (img_a - img_b).abs().max().item() > 1e-2
    # a list of PIL driver frames (the streaming path) after the switch
    pils = [FR.pil(ctx.size, 50 + i, "smooth") for i in range(2)]
    _, imgs = w.forward(ctx.src["B"], pils, crop=False, **BASE)
    _assert_match([imgs[0:1], imgs[1:2]], [fresh.forward(None, p, crop=False, **BASE)[1] for p in pils])
    assert captures[0] == 8     # and the fresh wrapper's four


def test_wrapper_identity_handle(ctx, captures, monkeypatch):
    """assigning A's handle back after B restores A's cached attributes and images, with no source pass and no capture"""
    from emoportraits_b200.infer import Model

    w = _wrapper(ctx)
    d = ctx.drv[1]
    pils = [FR.pil(ctx.size, 50 + i, "smooth") for i in range(2)]
    _, img_a = w.forward(ctx.src["A"], d, crop=False, **BASE)
    _, list_a = w.forward(None, pils, crop=False, **BASE)
    h_a = w.identity
    attrs_a = {k: getattr(w, k) for k in CACHED}
    _, img_b = w.forward(ctx.src["B"], d, crop=False, **BASE)
    assert w.identity is not h_a and not torch.equal(w.target_latent_volume, attrs_a["target_latent_volume"])
    passes = [0]
    orig = Model.source_pass

    def counted(self, *a, **k):
        passes[0] += 1
        return orig(self, *a, **k)

    monkeypatch.setattr(Model, "source_pass", counted)
    n = captures[0]
    w.identity = h_a
    assert w.identity is h_a
    for k in CACHED:
        assert torch.equal(getattr(w, k), attrs_a[k]), k
    _, img_a2 = w.forward(None, d, crop=False, **BASE)
    _, list_a2 = w.forward(None, pils, crop=False, **BASE)   # the list path animates A too
    assert passes[0] == 0 and captures[0] == n
    _assert_match([img_a2, list_a2[0:1], list_a2[1:2]], [img_a, list_a[0:1], list_a[1:2]])
    assert (img_a - img_b).abs().max().item() > 1e-2


def test_wrapper_smooth_pose_across_identity_switch(ctx, captures):
    """smooth_pose frames with reset_tracking on the first: A, then B through the same captured graph (loaded, not
    re-captured); each matches the eager smoothing recurrence on its own identity"""
    w = _wrapper(ctx)
    n_frames = 4

    def run(who):
        w.forward(ctx.src[who], None, crop=False, **BASE)
        return [w.forward(None, ctx.drv[i], crop=False, smooth_pose=True, reset_tracking=(i == 0), **BASE)[1]
                for i in range(n_frames)]

    def eager(st):
        state = torch.zeros((3, 4), device="cuda")
        return [w.model.driver_pass(st, ctx.drv[i], smooth_state=state, smooth_momentum=w.pose_momentum, smooth_init=(i == 0),
                                    **BASE)[0].clone() for i in range(n_frames)]

    got_a = run("A")
    st_a = w.identity
    assert captures[0] == 1
    got_b = run("B")
    assert captures[0] == 1
    _assert_match(got_a, eager(st_a))
    _assert_match(got_b, eager(w.identity))
    assert (got_a[-1] - got_b[-1]).abs().max().item() > 1e-2
