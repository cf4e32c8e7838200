"""CPU tests of identity switching (DriverPipeline.submit(..., st=), InferenceWrapper.identity, dist.new_identity):
  * in EMO_DRY_RUN mode, at 256^2 and 512^2 and for every pose option, Model.driver_pass on a graph's identity buffers
    issues the same launches, descriptor for descriptor, as on the source state they were loaded from, and reads the
    buffers' memory, not the state's;
  * the identity buffers and the broadcast state share one layout (dist.new_identity), with source_theta_dev a view;
  * DriverPipeline.submit(st=) and InferenceWrapper.identity refuse a state whose identity fields do not fit the model;
  * the pipeline's scratch sets are disjoint from the eager passes' set 0."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _fields(d):
    """(scalar fields and NULL-ness of the pointer fields, set of the non-NULL pointers) of a ctypes descriptor"""
    out, ptrs = [], set()
    for name, typ in d._fields_:
        v = getattr(d, name)
        if typ is C.c_void_p:
            out.append((name, bool(v)))
            if v:
                ptrs.add(v)
        else:
            out.append((name, v))
    return tuple(out), ptrs


def _recorder(L, monkeypatch):
    calls, ptrs = [], set()
    launch = L.call

    def call(name, *args):
        if args and hasattr(args[0], "_obj"):          # a descriptor passed by reference
            f, p = _fields(args[0]._obj)
            calls.append((name, f))
            ptrs.update(p)
        else:                                          # scalar arguments: device pointers are data_ptr() values
            big = {a for a in args if isinstance(a, int) and a > 1 << 20}
            ptrs.update(big)
            calls.append((name, tuple(a.value if isinstance(a, C.c_float) else "ptr" if a in big else a for a in args)))
        return launch(name, *args)

    monkeypatch.setattr(L, "call", call)
    return calls, ptrs


def _model(size, device="cpu"):
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    cfg = shipped_config(size)
    return cfg, Model(cfg, synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0), device)


def _loaded(cfg, st):
    from emoportraits_b200.dist import new_identity, source_state_shapes

    ident = new_identity(cfg, "cpu")
    for k in source_state_shapes(cfg):
        getattr(ident, k).copy_(getattr(st, k))
    return ident


OPTIONS = [dict(mix=True), dict(mix=False), dict(mix=True, target_theta=False), dict(mix=True, mix_old=True)]


@pytest.mark.parametrize("size", [256, 512])
def test_driver_pass_on_identity_buffers_issues_the_same_launches(dry, monkeypatch, size):
    cfg, model = _model(size)
    torch.manual_seed(0)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    ident = _loaded(cfg, st)
    calls, ptrs = _recorder(dry, monkeypatch)
    fields = ("target_latent_volume", "idt_embed", "pred_source_theta")
    to_buf = {getattr(st, k).data_ptr(): getattr(ident, k).data_ptr() for k in fields}
    bufs = set(to_buf.values())
    for kw in OPTIONS:
        calls.clear(); ptrs.clear()
        model.driver_pass(st, x, **kw)
        want, want_ptrs = list(calls), set(ptrs)
        calls.clear(); ptrs.clear()
        model.driver_pass(ident, x, **kw)
        assert want and calls == want, kw
        assert not (ptrs & set(to_buf)), kw                      # the buffers' pass never touches the state
        assert ptrs & bufs == {to_buf[p] for p in want_ptrs & set(to_buf)}, kw
    # the identity fields are what the driver pass reads: volume and idt embedding always, the theta through mix / target_theta
    calls.clear(); ptrs.clear()
    model.driver_pass(ident, x, mix=True, target_theta=False)
    assert ptrs >= bufs


def test_identity_buffers_share_the_broadcast_layout():
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.dist import check_identity, new_identity, source_state_shapes

    cfg = shipped_config(256)
    ident = new_identity(cfg, "cpu")
    for k, shp in source_state_shapes(cfg).items():
        t = getattr(ident, k)
        assert t.shape == shp and t.dtype == torch.float32 and t.is_contiguous() and not t.any()
    assert ident.source_theta_dev.shape == (4, 4)
    assert ident.source_theta_dev.data_ptr() == ident.pred_source_theta.data_ptr()   # a view: one copy loads both
    ident.pred_source_theta.fill_(3.0)
    assert torch.equal(ident.source_theta_dev, torch.full((4, 4), 3.0))
    check_identity(ident, cfg)


def _bad_states(cfg):
    from emoportraits_b200.dist import new_identity

    other = new_identity(cfg, "cpu")
    other.target_latent_volume = torch.zeros(1, cfg.D, cfg.S, cfg.S, cfg.C // 2)
    ncdhw = new_identity(cfg, "cpu")
    ncdhw.target_latent_volume = ncdhw.target_latent_volume.permute(0, 4, 1, 2, 3)
    half = new_identity(cfg, "cpu")
    half.idt_embed = half.idt_embed.half()
    missing = new_identity(cfg, "cpu")
    del missing.target_latent_volume
    flat = new_identity(cfg, "cpu")
    flat.pred_source_theta = flat.pred_source_theta[0]
    return {"channels": other, "ncdhw_volume": ncdhw, "fp16": half, "missing_volume": missing, "theta_4x4": flat, "none": None}


def test_submit_refuses_a_state_of_the_wrong_shapes():
    """the check runs before anything is queued (a DriverPipeline's slots need CUDA streams: a bare instance is enough here)"""
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import DriverPipeline

    cfg = shipped_config(256)
    pipe = DriverPipeline.__new__(DriverPipeline)
    pipe.model, pipe.st, pipe.n, pipe.depth, pipe.slots = SimpleNamespace(cfg=cfg), object(), 0, 1, []
    for name, bad in _bad_states(cfg).items():
        if bad is None:
            continue          # st=None is the current identity
        with pytest.raises(ValueError, match="identity"):
            pipe.submit(torch.zeros(1, 3, 256, 256), st=bad)
        assert pipe.n == 0, name


def test_identity_assignment_refuses_a_state_of_the_wrong_shapes():
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper

    for size in (256, 512):
        cfg = shipped_config(size)
        w = InferenceWrapper.__new__(InferenceWrapper)      # the constructor needs a device; the check does not
        torch.nn.Module.__init__(w)
        w.cfg, w._state = cfg, None
        for name, bad in _bad_states(cfg).items():
            with pytest.raises(ValueError, match="identity"):
                w.identity = bad
            assert w.identity is None, name
    from emoportraits_b200.dist import new_identity

    with pytest.raises(ValueError, match="handle"):   # the right shapes, but not from a wrapper's source pass
        w.identity = new_identity(cfg, "cpu")
    assert w.identity is None


def test_pipeline_scratch_sets_are_apart_from_the_eager_set():
    from emoportraits_b200 import ops
    from emoportraits_b200.infer import DriverPipeline

    eager = ops._SLOT
    assert eager == 0
    for depth in range(1, 9):
        slots = DriverPipeline.scratch_slots(depth)
        assert len(slots) == depth == len(set(slots))
        assert eager not in slots and all(isinstance(k, int) and k > 0 for k in slots)
