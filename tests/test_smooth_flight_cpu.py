"""CPU tests of smoothed frames in flight (Model.driver_pass(pose_only= / pose_in=), Model.pose_step, PoseTrack,
DriverPipeline(smooth=True), InferenceWrapper.forward(..., smooth_pose=True) with several frames):
  * in EMO_DRY_RUN mode, at 256^2 and 512^2 and for every pose option, a frame split at its pose step issues the plain
    frame's launches descriptor for descriptor, except its pose launch, which is followed by the pose step: a theta_in +
    smooth_state launch with mix = 0 and the momentum fields of ops.pose_desc;
  * a smoothing pipeline, captured and replayed with host stand-ins for CUDA graphs, streams and events: each frame
    replays its head, runs its pose step on the pose stream after the head and after its track's previous step, and
    replays its tail after the step; smooth_init is set on exactly the first frame of a track and after reset();
  * every refusal of a track happens before anything is queued;
  * forward routes smoothed lists and batches of more than one frame to the smoothing pipeline with the wrapper's own
    track (whose state is self.theta), and keeps single frames and custom embeddings on their routes."""
import contextlib
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_embedding_drive_cpu import _wrapper
from test_identity_switch_cpu import OPTIONS, _fields, _model


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _pose_fields(rec):
    return dict(rec[2])


def _recorder(L, monkeypatch, log):
    """every C-ABI call appended to `log` as ("launch", name, descriptor fields or args, the smooth_state / theta_in pointers)"""
    launch = L.call

    def call(name, *args):
        if args and hasattr(args[0], "_obj"):
            d = args[0]._obj
            ptrs = (getattr(d, "smooth_state", None), getattr(d, "theta_in", None)) if name == "emo_pose_theta" else None
            log.append(("launch", name, _fields(d)[0], ptrs))
        else:
            log.append(("launch", name, tuple("ptr" if isinstance(a, int) and a > 1 << 20 else
                                              a.value if isinstance(a, C.c_float) else a for a in args), None))
        return launch(name, *args)

    monkeypatch.setattr(L, "call", call)


def _launches(log, fn):
    log.clear()
    out = fn()
    return [e[:3] for e in log if e[0] == "launch"], out


def _split(name_fields):
    """index of the one emo_pose_theta launch"""
    idx = [i for i, e in enumerate(name_fields) if e[1] == "emo_pose_theta"]
    assert len(idx) == 1, idx
    return idx[0]


def _smooth_fields(rec, momentum, init):
    from emoportraits_b200 import ops

    f = _pose_fields(rec)
    want = ops.pose_desc(1, None, None, 1, 1, 1, theta_in=1, smooth_state=1, smooth_momentum=momentum, smooth_init=init)
    assert f["theta_in"] and not f["srt"] and not f["source_theta"] and f["mix"] == 0 and f["mix_old"] == 0
    assert f["smooth_state"] and f["theta_out"] and f["theta_warp"] and f["align2d"] and f["invert_warp"] == 0
    assert f["smooth_init"] == (1 if init else 0)
    assert f["smooth_momentum"] == want.smooth_momentum and f["smooth_one_minus"] == want.smooth_one_minus
    return f


@pytest.mark.parametrize("size", [256, 512])
def test_split_frame_launches(dry, monkeypatch, size):
    from emoportraits_b200.infer import Model

    cfg, model = _model(size)
    torch.manual_seed(0)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    pe = torch.rand(1, cfg.expr_channels)
    srt = torch.rand(1, 9) + 0.5
    log = []
    _recorder(dry, monkeypatch, log)
    state = torch.zeros(3, 4)
    pose = (torch.zeros(1, 4, 4), torch.zeros(1, 3, 4), torch.zeros(1, 2, 3))
    inputs = [dict(drv=x), dict(drv=x, custom_pose_embed=pe), dict(drv=x, custom_srt=srt),
              dict(drv=None, custom_srt=srt, custom_pose_embed=pe)]
    for kw in OPTIONS:
        for inp in inputs:
            inp = dict(inp)
            drv = inp.pop("drv")
            plain, _ = _launches(log, lambda: model.driver_pass(st, drv, **inp, **kw))
            k = _split(plain)
            sequential, _ = _launches(log, lambda: model.driver_pass(st, drv, smooth_state=state, smooth_momentum=0.9, **inp, **kw))
            assert sequential[:k] == plain[:k] and sequential[k + 1:] == plain[k + 1:], (kw, inp.keys())
            head, (_, _, _, so) = _launches(log, lambda: model.driver_pass(st, drv, pose_only=True, **inp, **kw))
            assert head == plain[:k + 1], (kw, inp.keys())            # the unsmoothed pose launch, with theta_out
            assert _pose_fields(head[-1])["theta_out"] and not _pose_fields(head[-1])["smooth_state"]
            assert tuple(so.pred_target_theta.shape) == (1, 4, 4) and so.target_pose_embed is None
            for m, init in ((0.9, False), (0.5, True), (0.1, False)):
                step, _ = _launches(log, lambda: Model.pose_step(so.pred_target_theta, state, m, init, pose))
                assert len(step) == 1
                _smooth_fields(step[0], m, init)
            tail, (_, _, _, so2) = _launches(log, lambda: model.driver_pass(st, drv, pose_in=pose, **inp, **kw))
            assert tail == plain[k + 1:], (kw, inp.keys())
            assert so2.pred_target_theta is pose[0]
            # the sequential frame's one smoothing launch is the split frame's pose launch and pose step
            assert head + step + tail == sequential[:k] + [plain[k]] + step + sequential[k + 1:]


def test_pose_in_refuses_other_pose_options(dry):
    _, model = _model(256)
    x = torch.rand(1, 3, 256, 256)
    st = model.source_pass(x)
    pose = (torch.zeros(1, 4, 4), torch.zeros(1, 3, 4), torch.zeros(1, 2, 3))
    for kw in (dict(pose_only=True), dict(smooth_state=torch.zeros(3, 4)), dict(pose_override=pose)):
        with pytest.raises(ValueError, match="pose_in"):
            model.driver_pass(st, x, pose_in=pose, **kw)
    with pytest.raises(ValueError, match="driver image"):        # an image-free tail still needs the embedding
        model.driver_pass(st, None, pose_in=pose)


# ---- a smoothing pipeline on host stand-ins -------------------------------------------------------------------------------
class _Cuda:
    """CUDA graphs, streams and events replaced by host stand-ins that append to one log; a graph keeps the launches issued
    while it was captured, and its replay logs them as one entry"""

    def __init__(self, monkeypatch, log):
        self.log, self.stack, self.n_streams, self.n_events = log, [], 0, 0
        cuda = self
        self.default = self.Stream()

        monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: cuda.Stream())
        monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: cuda.Event())
        monkeypatch.setattr(torch.cuda, "stream", self.stream)
        monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: self.current())
        monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
        monkeypatch.setattr(torch.cuda, "CUDAGraph", lambda: SimpleNamespace(launches=None, replay=None))
        monkeypatch.setattr(torch.cuda, "graph", self.graph)

    def current(self):
        return self.stack[-1] if self.stack else self.default

    @contextlib.contextmanager
    def stream(self, s):
        self.stack.append(s)
        try:
            yield
        finally:
            self.stack.pop()

    @contextlib.contextmanager
    def graph(self, g):
        start = len(self.log)
        yield
        g.launches = [e[:3] for e in self.log[start:] if e[0] == "launch"]
        del self.log[start:]
        g.replay = lambda: self.log.append(("replay", id(g), self.current().id))

    def Stream(self):
        cuda = self

        class S:
            def __init__(self):
                self.id = f"s{cuda.n_streams}"
                cuda.n_streams += 1

            def wait_stream(self, other):
                cuda.log.append(("wait_stream", self.id, other.id))

            def wait_event(self, ev):
                cuda.log.append(("wait_event", self.id, ev.id))

        return S()

    def Event(self):
        cuda = self

        class E:
            def __init__(self):
                self.id = f"e{cuda.n_events}"
                cuda.n_events += 1

            def record(self, *a):
                cuda.log.append(("record", self.id, cuda.current().id))

        return E()


@pytest.fixture(scope="module")
def model256():
    from emoportraits_b200 import lib as L

    mp = pytest.MonkeyPatch()
    mp.setattr(L, "DRY_RUN", True)
    try:
        cfg, model = _model(256)
        torch.manual_seed(1)
        st = model.source_pass(torch.rand(1, 3, 256, 256))
    finally:
        mp.undo()
    return cfg, model, st


def _smoothing_pipeline(dry, monkeypatch, model, st, depth=2, **kw):
    from emoportraits_b200.infer import DriverPipeline

    log = []
    _recorder(dry, monkeypatch, log)
    cuda = _Cuda(monkeypatch, log)
    pipe = DriverPipeline(model, st, depth=depth, smooth=True, **kw)
    log.clear()
    return pipe, log, cuda


def test_pipeline_frames_run_head_pose_step_tail(dry, monkeypatch, model256):
    cfg, model, st = model256
    x = torch.rand(1, 3, 256, 256)
    pipe, log, cuda = _smoothing_pipeline(dry, monkeypatch, model, st, depth=2, mix=True)
    # each slot's two graphs hold the split frame's launches
    plain, _ = _launches(log, lambda: model.driver_pass(st, x, mix=True))
    log.clear()
    k = _split(plain)
    for sl in pipe.slots:
        assert sl.run.head_graph.launches == plain[:k + 1] and sl.run.graph.launches == plain[k + 1:]
        with pytest.raises(RuntimeError, match="track"):
            sl.run(x)                       # a split frame is not a one-graph replay
    tracks = [pipe.track(momentum=m) for m in (0.9, 0.5, 0.1)]
    order = [0, 1, 0, 2, 2, 1, 0, 0, 1]     # frame i on track order[i]: interleaved, and runs of one track
    resets = {5: 1, 7: 0}                   # before frame 5, track 1 is reset; before frame 7, track 0
    for i, t in enumerate(order):
        if i in resets:
            tracks[resets[i]].reset()
        pipe.submit(x, track=tracks[t])
    # the pose steps, in submit order
    steps = [e for e in log if e[0] == "launch" and e[1] == "emo_pose_theta"]
    assert len(steps) == len(order) and not [e for e in log if e[0] == "launch" and e[1] != "emo_pose_theta"]
    seen = set()
    for i, (t, e) in enumerate(zip(order, steps)):
        sl = pipe.slots[i % pipe.depth]
        init = t not in seen or resets.get(i) == t
        seen.add(t)
        _smooth_fields(e, tracks[t].momentum, init)
        assert e[3] == (tracks[t].state.data_ptr(), sl.run.static_mixed.data_ptr()), i
    # per frame: head on the slot's stream, its event; the pose stream waits for it and for the track's previous step, runs
    # the step and records; the slot's stream waits for that and replays the tail
    pose = pipe.pose_stream.id
    last = {}
    pos = 0
    for i, t in enumerate(order):
        sl = pipe.slots[i % pipe.depth]
        s = sl.stream.id
        j = log.index(("replay", id(sl.run.head_graph), s), pos)
        head_ev = log[j + 1]
        assert head_ev[0] == "record" and head_ev[2] == s
        j += 2
        assert log[j] == ("wait_event", pose, head_ev[1])
        j += 1
        if t in last:
            assert log[j] == ("wait_event", pose, last[t])
            j += 1
        assert log[j][:2] == ("launch", "emo_pose_theta") and log[j] is steps[i]
        assert log[j + 1][0] == "record" and log[j + 1][2] == pose
        last[t] = log[j + 1][1]
        assert log[j + 2] == ("wait_event", s, last[t])
        assert log[j + 3] == ("replay", id(sl.run.graph), s)
        pos = j + 4
    assert all(tr.seeded for tr in tracks) and [tr.event.id for tr in tracks] == [last[t] for t in range(3)]


def test_momentum_is_read_at_submit(dry, monkeypatch, model256):
    cfg, model, st = model256
    x = torch.rand(1, 3, 256, 256)
    pipe, log, _ = _smoothing_pipeline(dry, monkeypatch, model, st, depth=1, mix=True)
    tr = pipe.track()
    for m in (0.5, 0.9, 0.3):
        tr.momentum = m
        pipe.submit(x, track=tr)
    steps = [e for e in log if e[0] == "launch" and e[1] == "emo_pose_theta"]
    for e, m, init in zip(steps, (0.5, 0.9, 0.3), (True, False, False)):
        _smooth_fields(e, m, init)
    # 0.9: fp32(1 - 0.9) is not 1 - fp32(0.9); the step passes the former, as pose_desc does
    f = _pose_fields(steps[1])
    assert f["smooth_one_minus"] == C.c_float(1.0 - 0.9).value != C.c_float(1.0 - C.c_float(0.9).value).value


def test_refusals_before_anything_is_queued(dry, monkeypatch, model256):
    from emoportraits_b200.infer import DriverPipeline, PoseTrack

    cfg, model, st = model256
    x = torch.rand(1, 3, 256, 256)
    pipe, log, cuda = _smoothing_pipeline(dry, monkeypatch, model, st, depth=1, mix=True)
    plain = DriverPipeline(model, st, depth=1, mix=True)
    log.clear()
    good = pipe.track()
    for m in (-0.1, 1.5, float("nan"), "x"):
        with pytest.raises(ValueError):
            pipe.track(momentum=m)
    other = PoseTrack("meta")
    bad_m = pipe.track()
    bad_m.momentum = 1.01
    cases = [(plain, dict(track=good)),                         # a track on a pipeline built without smooth
             (pipe, dict()),                                     # a smoothing pipeline's frame without a track
             (pipe, dict(track=other)),                          # a track on another device
             (pipe, dict(track=bad_m)),                          # a momentum outside [0, 1]
             (pipe, dict(track=SimpleNamespace(state=torch.zeros(3, 4), momentum=0.5, seeded=False, event=None)))]
    for p, kw in cases:
        n0, st0 = p.n, p.st
        with pytest.raises(ValueError):
            p.submit(x, st=st, **kw)
        assert p.n == n0 and p.st is st0 and not log, kw
    assert not good.seeded and good.event is None
    with pytest.raises(ValueError, match="encode"):
        DriverPipeline(SimpleNamespace(check_inputs=lambda *a: None, check_refine=lambda *a: None), None, depth=1,
                       encode=True, smooth=True)


# ---- InferenceWrapper.forward -----------------------------------------------------------------------------------------------
class _FakePipeline:
    def __init__(self, cfg, flags):
        self.flags, self.subs, self.depth = flags, [], 4
        so = SimpleNamespace(pred_target_theta=torch.full((1, 4, 4), 2.0), srt=torch.arange(9.0)[None],
                             target_pose_embed=torch.full((1, cfg.expr_channels), 3.0))
        self.slot = SimpleNamespace(run=SimpleNamespace(static_state=so))

    def submit(self, drv, **kw):
        self.subs.append(dict(kw, drv=drv, seeded=kw["track"].seeded if kw.get("track") else None))
        if kw.get("track"):
            kw["track"].seeded = True
        return SimpleNamespace(slot=self.slot)

    def drain(self):
        pass


def _routing_wrapper(monkeypatch):
    w = _wrapper()
    w._track = None
    pipes = []

    def pipeline(mix, target_theta, mix_old, **inputs):
        pipes.append(_FakePipeline(w.cfg, dict(mix=mix, target_theta=target_theta, mix_old=mix_old, **inputs)))
        return pipes[-1]

    rendered = []

    def render(pipe, n, inputs):
        subs = [inputs(i) for i in range(n)]
        for kw in subs:
            pipe.submit(**kw)
        rendered.append((pipe, subs))
        return [None] * n, torch.zeros(n, 3, 256, 256)

    monkeypatch.setattr(w, "_driver_pipeline", pipeline)
    monkeypatch.setattr(w, "_render", render)
    return w, pipes, rendered


def test_forward_routes_smoothed_lists_and_batches_to_the_pipeline(dry, monkeypatch):
    w, pipes, rendered = _routing_wrapper(monkeypatch)
    frames = [np.zeros((256, 256, 3), np.uint8) for _ in range(3)]
    w.forward(None, frames, crop=False, smooth_pose=True, mix=True, mix_old=False, reset_tracking=True)
    p, subs = rendered[-1]
    assert p.flags == dict(mix=True, target_theta=True, mix_old=False, theta_embed=False, pose_embed=False, smooth=True)
    tr = w._track
    assert len(subs) == 3 and all(s["track"] is tr for s in subs) and tr.state is w.theta
    assert [s["seeded"] for s in p.subs] == [False, True, True]           # the reset seeds on the first frame
    assert tr.momentum == w.pose_momentum
    # the next call carries the recurrence on: same track, same state, not re-seeded
    w.forward(None, frames, crop=False, smooth_pose=True)
    assert rendered[-1][0].subs[0]["track"] is tr and rendered[-1][0].subs[0]["seeded"] is True and tr.state is w.theta
    # a reset: the same state tensor, seeded again
    w.forward(None, frames[:2], crop=False, smooth_pose=True, reset_tracking=True)
    assert rendered[-1][0].subs[0]["track"] is tr and rendered[-1][0].subs[0]["seeded"] is False and tr.state is w.theta
    # a tensor batch of N > 1
    batch = torch.rand(3, 3, 256, 256)
    w.forward(None, batch, crop=False, smooth_pose=True)
    p = pipes[-1]
    assert p.flags["smooth"] and len(p.subs) == 3 and all(s["track"] is tr for s in p.subs)
    assert all(torch.equal(s["drv"], batch[i:i + 1]) and "dev_out" in s for i, s in enumerate(p.subs))
    assert torch.equal(w.pred_target_theta, torch.full((1, 4, 4), 2.0))
    assert torch.equal(torch.cat(w.pred_target_srt, 1), torch.arange(9.0)[None])
    # plain frames keep their pipeline and submit no track
    w.forward(None, batch, crop=False)
    assert "smooth" not in pipes[-1].flags and all("track" not in s for s in pipes[-1].subs)
    w.forward(None, frames, crop=False)
    assert "smooth" not in rendered[-1][0].flags and all("track" not in s for s in rendered[-1][1])
    # a momentum outside [0, 1] is refused before anything is queued
    n = len(pipes)
    w.pose_momentum = 1.5
    with pytest.raises(ValueError):
        w.forward(None, frames, crop=False, smooth_pose=True)
    assert len(pipes) == n


def test_forward_keeps_single_and_custom_smoothed_frames_on_their_routes(dry, monkeypatch):
    w, pipes, rendered = _routing_wrapper(monkeypatch)
    E = w.cfg.expr_channels
    seen = []

    def eager(st, drv, **kw):
        seen.append(kw)
        so = SimpleNamespace(pred_target_theta=torch.zeros(1, 4, 4), srt=torch.zeros(1, 9), target_pose_embed=torch.zeros(1, E))
        return torch.zeros(1, 3, 256, 256), None, None, so

    w.model = SimpleNamespace(driver_pass=eager)
    for one in (torch.rand(1, 3, 256, 256), [np.zeros((256, 256, 3), np.uint8)], np.zeros((256, 256, 3), np.uint8)):
        seen.clear()
        w.theta = None
        w.forward(None, one, crop=False, smooth_pose=True)   # the first smoothed frame seeds the state eagerly
        assert len(seen) == 1 and seen[0]["smooth_init"] and seen[0]["smooth_state"] is w.theta
    frames = [np.zeros((256, 256, 3), np.uint8) for _ in range(2)]
    seen.clear()
    w.forward(None, frames, crop=False, smooth_pose=True, reset_tracking=True, custome_target_pose_embed=torch.zeros(1, E))
    assert len(seen) == 2 and seen[0]["smooth_init"] and not seen[1]["smooth_init"]
    assert not pipes and not rendered
