"""CPU tests of composited, masked refined frames (Stage2Model.refine with stage 2's mask networks and a composite,
Model.make_driver_graph / DriverPipeline with refine_masks= and composite=, InferenceWrapper.forward_refined(bg=, mask_fn=),
emo_s2_prepare_composite / emo_s2_masked_stem / emo_s2_finish_masked):
  * in EMO_DRY_RUN mode, with the stand-in mask networks on the host, exact and fast stage 2 at 256^2 -> 512^2 and
    512^2 -> 1024^2, a composited, masked refined frame issues the stage-1 frame's launches, the compositing matte network's,
    emo_s2_prepare_composite, the stage-2 mask helpers' launches, emo_s2_masked_stem, the eager stage-2 convolutions
    (descriptor for descriptor) and emo_s2_finish_masked; without masks the launches are the unmasked refined frame's;
  * bad backgrounds, matte networks and stage-2 mask networks are refused before anything is queued;
  * a capture that a caller's network breaks raises the documented error, naming that network;
  * the three entry points refuse null pointers, bad shapes, a missing or doubled stem operand and misalignment."""
import contextlib
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from test_embedding_drive_cpu import _bare_pipeline, _identity
from test_identity_switch_cpu import _model
from test_identity_switch_cpu import _recorder as _desc_recorder
from test_refine_stream_cpu import _checker, _launches, _refining_wrapper, _s2_wrapper, _stage2

FAKE = 0x1000   # a 16-byte aligned non-null "device pointer" that is never dereferenced: the calls below are refused first


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _recorder(L, monkeypatch):
    """test_identity_switch_cpu's launch recorder, with the host arrays some entry points take (emo_parsing_masks' label
    sets) recorded as tuples of their values"""
    calls, ptrs = _desc_recorder(L, monkeypatch)
    record = L.call

    def call(name, *args):
        return record(name, *(tuple(a) if isinstance(a, C.Array) else a for a in args))

    monkeypatch.setattr(L, "call", call)
    return calls, ptrs


def _nets():
    """the stand-in networks on the host: (modnet, face_idt, the video loop's matte callable)"""
    from emoportraits_b200 import masks
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    modnet, face_idt = StubMODNet(), masks.FaceParsing(None, device="cpu", net=StubBiSeNet())
    return modnet, face_idt, masks.face_matte(face_idt, modnet)


@pytest.mark.parametrize("cloth", [False, True])
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("size,s2_size", [(256, 512), (512, 1024)])
def test_composited_masked_frame_launch_sequence(dry, monkeypatch, size, s2_size, precision, cloth):
    from emoportraits_b200 import masks

    _, model = _model(size)
    s2 = _stage2(s2_size, precision)
    modnet, face_idt, mask_fn = _nets()
    torch.manual_seed(0)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    bg = torch.rand(3, size, size)
    calls, _ = _recorder(dry, monkeypatch)
    frame = _launches(calls, lambda: model.driver_pass(st, x, mix=True))
    img = model.driver_pass(st, x, mix=True)[0]
    matte_calls = _launches(calls, lambda: mask_fn(img))
    resized = torch.rand(1, 3, s2_size, s2_size)
    helpers = _launches(calls, lambda: (masks.modnet_get_mask(modnet, resized), None if cloth else face_idt.label_masks(resized)))
    eager = _launches(calls, lambda: s2.forward(img, torch.rand(1, 1, s2_size, s2_size), None if cloth else torch.ones(1, 1, s2_size, s2_size)))
    skip = ["emo_resize_bilinear"] + (["emo_stem_pack"] if precision == "fast" else [])
    assert [c[0] for c in eager[:len(skip)]] == skip
    body = eager[len(skip):]

    def refined_frame():
        i = model.driver_pass(st, x, mix=True)[0]
        s2.refine(i, modnet=modnet, face_idt=face_idt, cloth=cloth, matte=mask_fn(i), bg=bg)

    got = _launches(calls, refined_frame)
    fast = precision == "fast"
    k = len(frame) + len(matte_calls)
    assert got[:len(frame)] == frame and got[len(frame):k] == matte_calls
    assert got[k] == ("emo_s2_prepare_composite", ("ptr", "ptr", "ptr", pytest.approx(0.3), 1, size, size, s2_size, "ptr", None, None,
                                                   0.0, 0)), got[k]
    assert got[k + 1:k + 1 + len(helpers)] == helpers
    k += 1 + len(helpers)
    assert got[k] == ("emo_s2_masked_stem", ("ptr", "ptr", 1, s2_size, None if fast else "ptr", "ptr" if fast else None,
                                             16.0 if fast else 0.0, 0)), got[k]
    assert got[k + 1:-1] == body
    assert got[-1] == ("emo_s2_finish_masked", ("ptr", "ptr", "ptr", None if cloth else "ptr", 1, s2_size, s2_size, "ptr", "ptr", 0))
    assert not {"emo_composite", "emo_image_to_u8", "emo_resize_bilinear", "emo_stem_pack"} & {c[0] for c in got[len(frame):]}


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_masks_without_composite_and_composite_without_masks(dry, monkeypatch, precision):
    s2 = _stage2(512, precision)
    modnet, face_idt, _ = _nets()
    img, bg, matte = torch.rand(1, 3, 256, 256), torch.rand(3, 256, 256), torch.rand(1, 1, 256, 256)
    calls, _ = _recorder(dry, monkeypatch)
    plain = _launches(calls, lambda: s2.refine(img))
    fast = precision == "fast"
    # the composite alone: the prepare pass writes the stem's operand, and the rest is the unmasked refined frame's
    comp = _launches(calls, lambda: s2.refine(img, matte=matte, bg=bg))
    assert comp[0][0] == "emo_s2_prepare_composite" and comp[0][1][9:12] == ((None, "ptr", 16.0) if fast else ("ptr", None, 0.0))
    assert comp[1:] == plain[1:]
    # the masks alone: emo_s2_prepare, then the masked stem overwrites its operand
    masked = _launches(calls, lambda: s2.refine(img, modnet=modnet, face_idt=face_idt))
    assert masked[0] == plain[0]
    assert [c[0] for c in masked].count("emo_s2_masked_stem") == 1 and masked[-1][0] == "emo_s2_finish_masked"


def test_refine_outputs_in_place_with_masks(dry):
    s2 = _stage2(512, "exact")
    modnet, face_idt, _ = _nets()
    out, u8 = torch.empty(1, 3, 512, 512), torch.empty(1, 512, 512, 3, dtype=torch.uint8)
    _, ffhq, got = s2.refine(torch.rand(1, 3, 256, 256), out=out, u8=u8, modnet=modnet, face_idt=face_idt,
                             matte=torch.rand(1, 1, 256, 256), bg=torch.rand(3, 256, 256))
    assert ffhq is out and got is u8


# ---- what is refused before anything is queued ------------------------------------------------------------------------------
def test_mask_networks_are_checked():
    from emoportraits_b200.infer import DriverPipeline, Model

    modnet, face_idt, mask_fn = _nets()
    refine = SimpleNamespace(device=torch.device("cpu"))
    Model.check_refine_masks(None)
    Model.check_refine_masks(refine, dict(modnet=modnet, face_idt=face_idt, cloth=True), mask_fn)
    bad = [(None, dict(modnet=modnet), None), (None, None, mask_fn),                          # no stage 2 to act on
           (refine, None, "not callable"), (refine, dict(modnet=modnet, extra=1), None),
           (refine, dict(modnet="not callable"), None), (refine, dict(face_idt=face_idt), None),   # a face mask needs the matte
           (refine, dict(modnet=modnet, face_idt=lambda x: x), None)]                           # not a FaceParsing
    for r, rm, comp in bad:
        with pytest.raises(ValueError):
            Model.check_refine_masks(r, rm, comp)
        with pytest.raises(ValueError):
            DriverPipeline(_checker(), None, depth=2, refine=r, refine_masks=rm, composite=comp)


def test_submit_refuses_bad_backgrounds():
    from emoportraits_b200.config import shipped_config

    cfg = shipped_config(256)
    img = torch.zeros(1, 3, 256, 256)
    cases = [(None, torch.zeros(3, 256, 256)),                                     # not a compositing pipeline
             (lambda x: x, None),                                                  # a compositing pipeline's frame needs one
             (lambda x: x, torch.zeros(3, 512, 512)), (lambda x: x, torch.zeros(1, 3, 256, 256)),
             (lambda x: x, torch.zeros(3, 256, 256, dtype=torch.float64)), (lambda x: x, [0.0] * 3)]
    for comp, bg in cases:
        pipe = _bare_pipeline(cfg, composite=comp)
        st0 = pipe.st
        with pytest.raises(ValueError, match="bg"):
            pipe.submit(img, bg=bg, st=SimpleNamespace(**vars(_identity(cfg))))
        assert pipe.n == 0 and pipe.st is st0


def test_forward_refined_refuses_bad_composites_and_networks(monkeypatch):
    w, seen = _refining_wrapper(monkeypatch)
    frames = torch.rand(2, 3, 256, 256)
    modnet, face_idt, mask_fn = _nets()
    s2 = _s2_wrapper()
    with_nets = lambda **kw: SimpleNamespace(**vars(_s2_wrapper()), **kw)    # noqa: E731
    bad = [dict(inferer_s2=s2, bg=torch.rand(3, 256, 256)),                    # a background without a matte network
           dict(inferer_s2=s2, mask_fn=mask_fn),                               # a matte network without a background
           dict(inferer_s2=s2, bg=torch.rand(3, 512, 512), mask_fn=mask_fn),
           dict(inferer_s2=s2, bg=torch.zeros(3, 256, 256, dtype=torch.uint8), mask_fn=mask_fn),
           dict(inferer_s2=s2, bg=torch.rand(3, 256, 256), mask_fn="not callable"),
           dict(inferer_s2=with_nets(modnet=None, face_idt=face_idt, cloth=False)),
           dict(inferer_s2=with_nets(modnet=modnet, face_idt=object(), cloth=False))]
    for kw in bad:
        with pytest.raises(ValueError):
            w.forward_refined(frames, **kw)
    assert not seen


def test_forward_refined_queues_composited_masked_frames(monkeypatch):
    w, seen = _refining_wrapper(monkeypatch)
    frames = torch.rand(3, 3, 256, 256)
    modnet, face_idt, mask_fn = _nets()
    s2 = SimpleNamespace(**vars(_s2_wrapper()), modnet=modnet, face_idt=face_idt, cloth=True)
    bg = torch.rand(3, 256, 256)
    w.forward_refined(frames, s2, bg=bg, mask_fn=mask_fn)
    flags, (_, subs) = seen[0], seen[1]
    assert flags["refine"] is s2.model_two and flags["composite"] is mask_fn
    assert flags["refine_masks"] == dict(modnet=modnet, face_idt=face_idt, cloth=True)
    assert len(subs) == 3 and all(torch.equal(s["bg"], bg) for s in subs) and all(s["bg"] is subs[0]["bg"] for s in subs)
    seen.clear()
    w.forward_refined(frames, _s2_wrapper())                                     # no networks, no composite: as before
    assert "refine_masks" not in seen[0] and "composite" not in seen[0] and "bg" not in seen[1][1][0]


# ---- a capture that a caller's network breaks ---------------------------------------------------------------------------------
def _fake_cuda(monkeypatch, capturing):
    """CUDA streams, events and graph capture replaced by host stand-ins; `capturing` is set inside the capture context"""
    stream = SimpleNamespace(wait_stream=lambda *a: None)

    @contextlib.contextmanager
    def graph(g):
        capturing.append(True)
        try:
            yield
        finally:
            capturing.clear()

    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: stream)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: stream)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", lambda: SimpleNamespace())
    monkeypatch.setattr(torch.cuda, "graph", graph)


@pytest.mark.parametrize("culprit", ["composite", "modnet", "face_idt"])
def test_capture_failure_names_the_network(dry, monkeypatch, culprit):
    cfg, model = _model(256)
    st = model.source_pass(torch.rand(1, 3, 256, 256))
    s2 = _stage2(512, "exact")
    modnet, face_idt, _ = _nets()
    mask_fn = _nets()[2]          # the compositing matte runs networks of its own
    capturing = []
    _fake_cuda(monkeypatch, capturing)

    def breaks_capture(fn):
        def call(*a, **k):
            if capturing:
                raise RuntimeError("operation not permitted when stream is capturing")
            return fn(*a, **k)
        return call

    if culprit == "composite":
        mask_fn = breaks_capture(mask_fn)
    elif culprit == "modnet":
        modnet = breaks_capture(modnet)
    else:
        face_idt.net = breaks_capture(face_idt.net)
    name = {"composite": "mask_fn", "modnet": "modnet", "face_idt": "face_idt"}[culprit]
    net_before = face_idt.net
    with pytest.raises(RuntimeError, match=name) as e:
        model.make_driver_graph(st, slot=1, refine=s2, refine_masks=dict(modnet=modnet, face_idt=face_idt), composite=mask_fn)
    assert "stage2.InferenceWrapper.forward" in str(e.value) and "host syncs" in str(e.value)
    assert isinstance(e.value.__cause__, RuntimeError) and "capturing" in str(e.value.__cause__)
    assert face_idt.net is net_before                  # the caller's face parser is left as it was: the capture wraps a copy
    # without a failure the same capture goes through, and the background buffer is the frame's
    if culprit == "composite":
        run = model.make_driver_graph(st, slot=1, refine=s2, refine_masks=dict(modnet=modnet), composite=_nets()[2])
        assert tuple(run.static_bg.shape) == (3, 256, 256) and run.static_u8 is not None


def test_capture_failure_elsewhere_is_not_blamed_on_a_network(dry, monkeypatch):
    _, model = _model(256)
    st = model.source_pass(torch.rand(1, 3, 256, 256))
    s2 = _stage2(512, "exact")
    modnet, face_idt, mask_fn = _nets()
    capturing = []
    _fake_cuda(monkeypatch, capturing)

    def refine(*a, **k):
        raise ValueError("a project error")

    monkeypatch.setattr(s2, "refine", refine)
    with pytest.raises(ValueError, match="a project error"):
        model.make_driver_graph(st, slot=1, refine=s2, refine_masks=dict(modnet=modnet), composite=mask_fn)


def test_composite_matte_shape_is_checked(dry, monkeypatch):
    _, model = _model(256)
    st = model.source_pass(torch.rand(1, 3, 256, 256))
    _fake_cuda(monkeypatch, [])
    with pytest.raises(ValueError, match=r"matte \(1,1,256,256\)"):
        model.make_driver_graph(st, slot=1, refine=_stage2(512, "exact"), composite=lambda img: torch.zeros(1, 3, 256, 256))


# ---- the entry points' argument checks ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from emoportraits_b200 import lib as L

    if L.DRY_RUN:
        pytest.skip("EMO_DRY_RUN skips the calls")
    L.load()
    return L


def _refused(lib, rc, match):
    assert rc == -1, rc                                  # EMO_ERR_INVALID
    msg = lib.emo_last_error().decode()
    assert match in msg, msg


def test_s2_prepare_composite_guards(L):
    lib = L.load()
    f = lambda *a: lib.emo_s2_prepare_composite(*a, None)   # noqa: E731
    for k in range(4):
        ptrs = [FAKE] * 4
        ptrs[k] = None
        _refused(lib, f(ptrs[0], ptrs[1], ptrs[2], 0.3, 1, 256, 256, 512, ptrs[3], FAKE, None, 0.0), "null pointer")
    _refused(lib, f(FAKE, FAKE, FAKE, 0.3, 1, 256, 256, 512, FAKE, FAKE, FAKE, 16.0), "at most one stem operand")
    for shape in ((0, 256, 256, 512), (1, 0, 256, 512), (1, 256, 0, 512), (1, 256, 256, 0)):
        _refused(lib, f(FAKE, FAKE, FAKE, 0.3, *shape, FAKE, None, None, 0.0), "bad shape")
    for k in range(4):
        ptrs = [FAKE] * 4
        ptrs[k] = FAKE + 2
        _refused(lib, f(ptrs[0], ptrs[1], ptrs[2], 0.3, 1, 256, 256, 512, ptrs[3], None, None, 0.0), "4-byte aligned")
    _refused(lib, f(FAKE, FAKE, FAKE, 0.3, 1, 256, 256, 512, FAKE, None, FAKE + 8, 16.0), "16-byte aligned")
    _refused(lib, f(FAKE, FAKE, FAKE, 0.3, 1, 256, 256, 512, FAKE, FAKE + 4, None, 0.0), "16-byte aligned")
    _refused(lib, f(FAKE, FAKE, FAKE, 0.3, 1, 256, 256, 512, FAKE, None, FAKE, 0.0), "plane_scale")
    _refused(lib, f(FAKE, FAKE, FAKE, 0.3, 1 << 20, 256, 256, 1 << 12, FAKE, None, None, 0.0), "grid too large")


def test_s2_masked_stem_guards(L):
    lib = L.load()
    f = lambda *a: lib.emo_s2_masked_stem(*a, None)   # noqa: E731
    _refused(lib, f(None, FAKE, 1, 512, FAKE, None, 0.0), "null pointer")
    _refused(lib, f(FAKE, None, 1, 512, FAKE, None, 0.0), "null pointer")
    _refused(lib, f(FAKE, FAKE, 1, 512, None, None, 0.0), "exactly one stem operand")
    _refused(lib, f(FAKE, FAKE, 1, 512, FAKE, FAKE, 16.0), "exactly one stem operand")
    for shape in ((0, 512), (1, 0)):
        _refused(lib, f(FAKE, FAKE, *shape, FAKE, None, 0.0), "bad shape")
    _refused(lib, f(FAKE + 2, FAKE, 1, 512, FAKE, None, 0.0), "4-byte aligned")
    _refused(lib, f(FAKE, FAKE + 2, 1, 512, FAKE, None, 0.0), "4-byte aligned")
    _refused(lib, f(FAKE, FAKE, 1, 512, None, FAKE + 8, 16.0), "16-byte aligned")
    _refused(lib, f(FAKE, FAKE, 1, 512, FAKE + 4, None, 0.0), "16-byte aligned")
    _refused(lib, f(FAKE, FAKE, 1, 512, None, FAKE, 0.0), "plane_scale")
    _refused(lib, f(FAKE, FAKE, 1 << 20, 1 << 12, FAKE, None, 0.0), "grid too large")


def test_s2_finish_masked_guards(L):
    lib = L.load()
    f = lambda *a: lib.emo_s2_finish_masked(*a, None)   # noqa: E731
    for k in range(5):
        ptrs = [FAKE] * 5
        ptrs[k] = None
        _refused(lib, f(ptrs[0], ptrs[1], ptrs[2], FAKE, 1, 512, 512, ptrs[3], ptrs[4]), "null pointer")
    for shape in ((0, 512, 512), (1, 0, 512), (1, 512, 0)):
        _refused(lib, f(FAKE, FAKE, FAKE, None, *shape, FAKE, FAKE), "bad shape")
    for k in range(4):
        ptrs = [FAKE] * 4
        ptrs[k] = FAKE + 1
        _refused(lib, f(ptrs[0], ptrs[1], ptrs[2], None, 1, 512, 512, ptrs[3], FAKE), "4-byte aligned")
