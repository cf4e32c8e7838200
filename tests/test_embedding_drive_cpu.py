"""CPU tests of driving frames from pose and expression embeddings (Model.driver_pass with drv=None / encode_only,
DriverPipeline's image / theta_embed / pose_embed / encode inputs, InferenceWrapper.encode / animate and forward with
custome_target_theta_embed / custome_target_pose_embed):
  * in EMO_DRY_RUN mode, at 256^2 and 512^2 and for every pose option, an image-free frame issues exactly the driver frame's
    launches without the head-pose regressor and the expression encoder, descriptor for descriptor; a frame with a custom
    embedding drops only the expression encoder, and an encoding frame is the driver frame's launches up to the encoder;
  * forward with a custom pose or embedding (and no smooth_pose) goes through a captured pipeline taking them as inputs,
    for a tensor batch and for a list of frames, and no longer calls the eager Model.driver_pass;
  * inputs other than a pipeline's, tensors of the wrong shape, mismatched counts and a missing source pass raise before
    anything is queued."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_identity_switch_cpu import OPTIONS, _model, _recorder


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _launches(calls, fn):
    calls.clear()
    fn()
    return list(calls)


@pytest.mark.parametrize("size", [256, 512])
def test_frame_launches_by_inputs(dry, monkeypatch, size):
    cfg, model = _model(size)
    torch.manual_seed(0)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    srt, pe = torch.rand(1, 9) + 0.5, torch.rand(1, cfg.expr_channels)
    calls, _ = _recorder(dry, monkeypatch)
    head = _launches(calls, lambda: model.head_pose_regressor(x))
    align = torch.zeros(1, 2, 3)
    encoder = _launches(calls, lambda: model.expression_embedder_nw(x, align))
    assert head and encoder
    for kw in OPTIONS:
        full = _launches(calls, lambda: model.driver_pass(st, x, **kw))
        assert full[:len(head)] == head, kw
        pose = full[len(head)]
        assert pose[0] == "emo_pose_theta", kw
        assert full[len(head) + 1:len(head) + 1 + len(encoder)] == encoder, kw
        rest = full[len(head) + 1 + len(encoder):]
        assert rest, kw
        free = _launches(calls, lambda: model.driver_pass(st, None, custom_srt=srt, custom_pose_embed=pe, **kw))
        assert free == [pose] + rest, kw
        assert _launches(calls, lambda: model.driver_pass(st, x, custom_pose_embed=pe, **kw)) == head + [pose] + rest, kw
        assert _launches(calls, lambda: model.driver_pass(st, x, custom_srt=srt, **kw)) == full, kw   # the regressed pose is kept
        assert _launches(calls, lambda: model.driver_pass(st, x, encode_only=True, **kw)) == full[:len(head) + 1 + len(encoder)], kw
    # the image-free frame reports the supplied pose and embedding
    _, _, _, so = model.driver_pass(st, None, custom_srt=srt, custom_pose_embed=pe, mix=True)
    assert torch.equal(so.srt, srt) and torch.equal(so.target_pose_embed, pe)


def test_driver_pass_without_an_image_needs_both_embeddings(dry):
    cfg, model = _model(256)
    st = model.source_pass(torch.rand(1, 3, 256, 256))
    srt, pe = torch.ones(1, 9), torch.zeros(1, cfg.expr_channels)
    for kw in (dict(custom_srt=srt), dict(custom_pose_embed=pe), {}, dict(custom_srt=srt, custom_pose_embed=pe, encode_only=True)):
        with pytest.raises(ValueError, match="driver image"):
            model.driver_pass(st, None, **kw)


# ---- inputs a captured frame takes ----------------------------------------------------------------------------------------
def test_input_sets():
    from emoportraits_b200.infer import DriverPipeline, Model

    ok = [dict(image=True), dict(image=True, theta_embed=True), dict(image=True, pose_embed=True),
          dict(image=True, theta_embed=True, pose_embed=True), dict(image=False, theta_embed=True, pose_embed=True),
          dict(image=True, encode=True)]
    bad = [dict(image=False), dict(image=False, theta_embed=True), dict(image=False, pose_embed=True),
           dict(image=True, encode=True, pose_embed=True), dict(image=True, encode=True, theta_embed=True),
           dict(image=False, theta_embed=True, pose_embed=True, encode=True)]
    full = dict(image=True, theta_embed=False, pose_embed=False, encode=False)
    for kw in ok:
        Model.check_inputs(**dict(full, **kw))
    for kw in bad:
        with pytest.raises(ValueError):
            Model.check_inputs(**dict(full, **kw))
        # the pipeline refuses the set before it creates a stream or captures anything
        with pytest.raises(ValueError):
            DriverPipeline(SimpleNamespace(check_inputs=Model.check_inputs), None, depth=4, **kw)


def _bare_pipeline(cfg, **inputs):
    """a DriverPipeline without slots (they need CUDA streams): enough for the checks, which run before anything is queued"""
    from emoportraits_b200.infer import DriverPipeline

    pipe = DriverPipeline.__new__(DriverPipeline)
    pipe.model, pipe.st, pipe.n, pipe.depth, pipe.slots = SimpleNamespace(cfg=cfg), object(), 0, 1, []
    pipe.image, pipe.theta_embed, pipe.pose_embed, pipe.encode = True, False, False, False
    vars(pipe).update(inputs)
    return pipe


def test_submit_refuses_other_inputs_and_shapes():
    from emoportraits_b200.config import shipped_config

    cfg = shipped_config(256)
    E = cfg.expr_channels
    img, srt, pe = torch.zeros(1, 3, 256, 256), torch.ones(1, 9), torch.zeros(1, E)
    cases = {
        "image": (dict(), [dict(drv=None), dict(drv=img, theta_embed=srt), dict(drv=img, pose_embed=pe)]),
        "theta": (dict(theta_embed=True), [dict(drv=img), dict(drv=img, theta_embed=srt, pose_embed=pe),
                                            dict(drv=img, theta_embed=torch.ones(9)), dict(drv=img, theta_embed=torch.ones(1, 3)),
                                            dict(drv=img, theta_embed=[1.0] * 9), dict(drv=None, theta_embed=srt)]),
        "pose": (dict(pose_embed=True), [dict(drv=img), dict(drv=img, pose_embed=torch.zeros(1, E - 1)),
                                          dict(drv=img, pose_embed=torch.zeros(2, E)), dict(drv=img, theta_embed=srt, pose_embed=pe)]),
        "image_free": (dict(image=False, theta_embed=True, pose_embed=True),
                       [dict(drv=img, theta_embed=srt, pose_embed=pe), dict(drv=None, theta_embed=srt),
                        dict(drv=None, pose_embed=pe), dict(drv=None, theta_embed=torch.ones(2, 9), pose_embed=torch.zeros(2, E)),
                        dict(drv=None, theta_embed=srt, pose_embed=pe.reshape(E))]),
        "encode": (dict(encode=True), [dict(drv=img, dev_out=img), dict(drv=img, host_out=img), dict(drv=None),
                                        dict(drv=img, pose_embed=pe)]),
    }
    for name, (inputs, bad) in cases.items():
        pipe = _bare_pipeline(cfg, **inputs)
        st0 = pipe.st
        for kw in bad:
            kw = dict(kw)
            with pytest.raises(ValueError):
                pipe.submit(kw.pop("drv"), st=SimpleNamespace(**vars(_identity(cfg))), **kw)
            assert pipe.n == 0 and pipe.st is st0, (name, kw)     # nothing queued, the identity not switched


def _identity(cfg):
    from emoportraits_b200.dist import new_identity

    return new_identity(cfg, "cpu")


# ---- InferenceWrapper -------------------------------------------------------------------------------------------------
def _wrapper(size=256, state=True):
    """an InferenceWrapper on the host (the constructor needs a device; the paths tested here do not)"""
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper

    w = InferenceWrapper.__new__(InferenceWrapper)
    torch.nn.Module.__init__(w)
    w.cfg, w.device, w._state = shipped_config(size), torch.device("cpu"), (_identity(shipped_config(size)) if state else None)
    w.theta, w.pose_momentum, w._smooth_graph = None, 0.5, None

    def eager(*a, **k):
        raise AssertionError("the eager driver pass was called")

    w.model = SimpleNamespace(driver_pass=eager)
    return w


class _FakePipeline:
    """records what the wrapper submits; its frames 'return' a fixed static state"""

    def __init__(self, cfg, **flags):
        self.flags, self.subs, self.depth = flags, [], 4
        so = SimpleNamespace(pred_target_theta=torch.full((1, 4, 4), 2.0), srt=torch.arange(9.0)[None],
                             target_pose_embed=torch.full((1, cfg.expr_channels), 3.0))
        self.slot = SimpleNamespace(run=SimpleNamespace(static_state=so))

    def submit(self, drv, **kw):
        self.subs.append(dict(kw, drv=drv))
        return SimpleNamespace(slot=self.slot)

    def drain(self):
        pass


def test_forward_with_custom_embeddings_is_captured(dry, monkeypatch):
    w = _wrapper()
    E = w.cfg.expr_channels
    pipes = []

    def pipeline(mix, target_theta, mix_old, **inputs):
        pipes.append(_FakePipeline(w.cfg, mix=mix, target_theta=target_theta, mix_old=mix_old, **inputs))
        return pipes[-1]

    monkeypatch.setattr(w, "_driver_pipeline", pipeline)
    srt = (torch.ones(1, 3), torch.full((1, 3), 0.1), torch.full((1, 3), 0.2))
    pe = torch.linspace(-1, 1, E)          # the eager path took any shape with E elements: so does this one
    drv = torch.rand(3, 3, 256, 256)
    for kw, flags in [(dict(custome_target_theta_embed=srt), dict(theta_embed=True, pose_embed=False)),
                      (dict(custome_target_pose_embed=pe), dict(theta_embed=False, pose_embed=True)),
                      (dict(custome_target_theta_embed=srt, custome_target_pose_embed=pe), dict(theta_embed=True, pose_embed=True))]:
        pil, img = w.forward(None, drv, crop=False, mix=True, mix_old=False, **kw)
        p = pipes[-1]
        assert p.flags == dict(mix=True, target_theta=True, mix_old=False, **flags)
        assert len(p.subs) == 3 and len(pil) == 3 and img.shape == (3, 3, 256, 256)
        for i, s in enumerate(p.subs):
            assert torch.equal(s["drv"], drv[i:i + 1]) and s["st"] is w._state
            want_srt = torch.cat(srt, 1) if flags["theta_embed"] else None
            want_pe = pe.reshape(1, E) if flags["pose_embed"] else None
            for k, want in (("theta_embed", want_srt), ("pose_embed", want_pe)):
                assert (s[k] is None) if want is None else torch.equal(s[k], want), (kw.keys(), k)
        # the attributes come from the captured frame: pred_target_srt is its (regressed) pose
        assert torch.equal(torch.cat(w.pred_target_srt, 1), torch.arange(9.0)[None])
        assert torch.equal(w.target_pose_embed, torch.full((1, E), 3.0))
    # a list of frames takes the streaming path, with the same inputs for every frame
    seen = []
    monkeypatch.setattr(w, "_render", lambda pipe, n, inputs: seen.append((pipe, [inputs(i) for i in range(n)])))
    frames = [np.zeros((256, 256, 3), np.uint8) for _ in range(3)]
    w.forward(None, frames, crop=False, mix=True, custome_target_pose_embed=pe)
    pipe, subs = seen[-1]
    assert pipe.flags["pose_embed"] and not pipe.flags["theta_embed"] and len(subs) == 3
    assert all(s["theta_embed"] is None and torch.equal(s["pose_embed"], pe.reshape(1, E)) and s["drv"].shape == (1, 3, 256, 256)
               for s in subs)


def test_smooth_pose_with_custom_embedding_stays_eager(dry, monkeypatch):
    w = _wrapper()
    E = w.cfg.expr_channels
    monkeypatch.setattr(w, "_driver_pipeline", lambda *a, **k: pytest.fail("no pipeline for smooth_pose"))
    seen = []

    def eager(st, drv, **kw):
        seen.append(kw)
        so = SimpleNamespace(pred_target_theta=torch.zeros(1, 4, 4), srt=torch.zeros(1, 9), target_pose_embed=torch.zeros(1, E))
        return torch.zeros(1, 3, 256, 256), None, None, so

    w.model = SimpleNamespace(driver_pass=eager)
    w.forward(None, torch.rand(2, 3, 256, 256), crop=False, smooth_pose=True, custome_target_pose_embed=torch.zeros(1, E))
    assert len(seen) == 2 and seen[0]["smooth_init"] and not seen[1]["smooth_init"]
    assert seen[0]["custom_pose_embed"] is not None


def test_animate_and_encode_refuse_before_queueing(monkeypatch):
    w = _wrapper()
    E = w.cfg.expr_channels
    monkeypatch.setattr(w, "_driver_pipeline", lambda *a, **k: pytest.fail("queued"))
    three = lambda n: (torch.ones(n, 3), torch.zeros(n, 3), torch.zeros(n, 3))   # noqa: E731
    bad = [
        (three(4), torch.zeros(5, E)),                                # mismatched N
        ((torch.ones(4, 3), torch.zeros(3, 3), torch.zeros(4, 3)), torch.zeros(4, E)),
        (three(4), torch.zeros(4, E + 1)),                            # wrong embedding size
        (three(4), torch.zeros(4 * E)),
        ((torch.ones(4, 9),), torch.zeros(4, E)),                     # not (scale, rotation, translation)
        (torch.ones(4, 9), torch.zeros(4, E)),
        ((torch.ones(4, 1, 3), torch.zeros(4, 3), torch.zeros(4, 3)), torch.zeros(4, E)),
        (three(0), torch.zeros(0, E)),                                # no frame
    ]
    for theta, pe in bad:
        with pytest.raises(ValueError):
            w.animate(theta, pe)
    none = _wrapper(state=False)
    monkeypatch.setattr(none, "_driver_pipeline", lambda *a, **k: pytest.fail("queued"))
    with pytest.raises(RuntimeError, match="source"):
        none.animate(three(2), torch.zeros(2, E))
    with pytest.raises(RuntimeError, match="source"):
        none.encode(torch.zeros(2, 3, 256, 256))
