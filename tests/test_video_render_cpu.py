"""CPU tests of the device-side video loop (ops.resample_u8 / ops.mask_dilate, video.get_bg, video.render_video):
  * ops.resample_coeffs drives a numpy restatement of emo_resample_u8's two integer passes, which must equal the installed
    Pillow's Image.crop(box).resize(size, f) bit for bit: LANCZOS and BICUBIC, up and down, odd sizes, 1024 -> 512,
    1920x1080 -> 512, and boxes inside the image, partly outside it, around it and fully outside it (Pillow's zero padding);
  * in EMO_DRY_RUN mode render_video and get_bg issue the documented launches per frame, reuse a bounded ring of row
    buffers, and refuse bad inputs before anything is queued."""
import contextlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

FILTERS = {"lanczos": Image.LANCZOS, "bicubic": Image.BICUBIC}

# (source height, width, crop box or None, output (width, height)): the grid the device kernel is held to as well
RESAMPLE_CASES = [
    (64, 80, None, (37, 29)),                       # down, odd sizes
    (41, 37, None, (100, 77)),                      # up, odd sizes
    (50, 60, None, (60, 31)),                       # vertical pass only
    (50, 60, None, (17, 50)),                       # horizontal pass only
    (50, 60, None, (60, 50)),                       # same size: a copy
    (1024, 1024, None, (512, 512)),                 # the video row's output panel
    (1080, 1920, None, (512, 512)),                 # a decoded 1080p frame to the driver frame
    (512, 512, (64, 80, 448, 400), (512, 512)),     # the notebook's fixed crop, back to the frame size
    (300, 260, (-40, -25, 200, 180), (150, 170)),   # partly outside
    (120, 100, (-30, -20, 140, 150), (90, 85)),     # around the whole image
    (120, 100, (130, 10, 170, 60), (33, 21)),       # fully outside: zeros
    (120, 100, (10, 20, 60, 70), (50, 50)),         # a crop at its own size: a copy of the crop
]


def _crop(a, box):
    """Image.crop: pixels outside the source are 0"""
    H, W = a.shape[:2]
    x0, y0, x1, y1 = box
    out = np.zeros((y1 - y0, x1 - x0, 3), np.uint8)
    sy0, sy1, sx0, sx1 = max(y0, 0), min(y1, H), max(x0, 0), min(x1, W)
    if sy1 > sy0 and sx1 > sx0:
        out[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = a[sy0:sy1, sx0:sx1]
    return out


def _pass(a, taps):
    """one horizontal pass of emo_resample_u8 over rows of a (H, W, 3): int32 sums from 1 << 21, >> 22, clipped"""
    out = np.empty((a.shape[0], len(taps), 3), np.uint8)
    for x, (first, k) in enumerate(taps):
        acc = np.full((a.shape[0], 3), 1 << 21, np.int64)
        for j, kk in enumerate(k):
            acc += a[:, first + j].astype(np.int64) * kk
        assert np.abs(acc).max() < 2 ** 31             # the kernel's int32 sums cannot overflow
        out[:, x] = np.clip(acc >> 22, 0, 255)
    return out


def np_resample(a, size, filt, box=None):
    """the two passes of emo_resample_u8, in numpy, driven by ops.resample_coeffs"""
    from emoportraits_b200 import ops

    c = _crop(a, box or (0, 0, a.shape[1], a.shape[0]))
    ch, cw = c.shape[:2]
    ow, oh = size
    ht = ops.resample_coeffs(cw, ow, filt) if ow != cw else None
    vt = ops.resample_coeffs(ch, oh, filt) if oh != ch else None
    if ht is not None:
        if vt is not None:
            lo, hi = vt[0][0], vt[-1][0] + len(vt[-1][1])   # the rows the vertical pass reads
            c, vt = _pass(c[lo:hi], ht), [(f - lo, k) for f, k in vt]
        else:
            c = _pass(c, ht)
    if vt is not None:
        c = _pass(c.transpose(1, 0, 2), vt).transpose(1, 0, 2)
    return c


def pil_resample(a, size, filt, box=None):
    im = Image.fromarray(a)
    return np.asarray((im.crop(box) if box is not None else im).resize(size, FILTERS[filt]))


@pytest.mark.parametrize("filt", sorted(FILTERS))
@pytest.mark.parametrize("case", range(len(RESAMPLE_CASES)))
def test_coefficient_tables_reproduce_pillow(filt, case):
    H, W, box, size = RESAMPLE_CASES[case]
    a = np.random.default_rng(case).integers(0, 256, (H, W, 3), dtype=np.uint8)
    assert np.array_equal(np_resample(a, size, filt, box), pil_resample(a, size, filt, box))


def test_tables_are_cached_with_pillows_ybox():
    from emoportraits_b200 import ops

    t = ops.resample_taps(1080, 512, "bicubic", "cpu")
    assert ops.resample_taps(1080, 512, "bicubic", "cpu") is t
    coeffs = ops.resample_coeffs(1080, 512, "bicubic")
    assert t.table.dtype == torch.int32 and tuple(t.table.shape) == (512, 2 + t.kmax)
    assert (t.lo, t.hi) == (coeffs[0][0], coeffs[-1][0] + len(coeffs[-1][1]))
    assert t.table[7, 0] == coeffs[7][0] and t.table[7, 1] == len(coeffs[7][1])
    with pytest.raises(ValueError):
        ops.resample_taps(10, 5, "bilinear", "cpu")


# ---- render_video / get_bg on the host (EMO_DRY_RUN) ----------------------------------------------------------------------
class _Event:
    log = []

    def __init__(self):
        self.id = len([e for e in _Event.log if e[0] == "new"])
        _Event.log.append(("new", self.id))

    def record(self, *a):
        _Event.log.append(("record", self.id))

    def synchronize(self):
        _Event.log.append(("sync", self.id))


class _Writer:
    instances = []

    def __init__(self, path, fourcc, fps, dims):
        self.args, self.rows, self.released = (path, fps, dims), [], False
        _Writer.instances.append(self)

    def write(self, row):
        self.rows.append(row)

    def release(self):
        self.released = True


class _Pipe:
    def __init__(self, depth, s2):
        self.depth, self.subs, self.drained = depth, [], 0
        self.slot = SimpleNamespace(stream="slot-stream", run=SimpleNamespace(static_u8=torch.zeros(1, s2, s2, 3, dtype=torch.uint8)))

    def submit(self, drv, **kw):
        self.subs.append(dict(kw, drv=drv))
        return SimpleNamespace(slot=self.slot, done=None)

    def drain(self):
        self.drained += 1


@pytest.fixture
def host(monkeypatch):
    """EMO_DRY_RUN with CUDA streams, events, pinned memory and cv2.VideoWriter replaced by host stand-ins; the launches are
    recorded as (name, args) with pointers as 'ptr' / None"""
    import cv2

    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: "current-stream")
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    monkeypatch.setattr(cv2, "VideoWriter", _Writer)
    _Event.log, _Writer.instances = [], []
    calls = []
    record = L.call

    def call(name, *args):
        calls.append((name, tuple("ptr" if isinstance(a, int) and a > 1 << 20 else a for a in args[:-1])))
        return record(name, *args)

    monkeypatch.setattr(L, "call", call)
    return calls


def _inferer(monkeypatch, depth=4, s2=512, state=True):
    from test_refine_stream_cpu import _refining_wrapper

    w, seen = _refining_wrapper(monkeypatch, state=state)
    pipe = _Pipe(depth, s2)

    def pipeline(mix, target_theta, mix_old, refine=None, **inputs):
        seen.append(dict(mix=mix, target_theta=target_theta, mix_old=mix_old, refine=refine, **inputs))
        return pipe

    monkeypatch.setattr(w, "_driver_pipeline", pipeline)
    return w, pipe, seen


def _pils(n, size=256, mode="RGB"):
    rng = np.random.default_rng(n)
    return [Image.fromarray(rng.integers(0, 256, (size, size, 3), dtype=np.uint8)).convert(mode) for _ in range(n)]


def _shape(call):
    """an emo_resample_u8 call as (source h, w, bgr, crop x0, y0, w, h, out h, w, dst bgr, horizontal taps?, vertical taps?)"""
    a = call[1]
    return (a[1], a[2], a[4], a[5], a[6], a[7], a[8], a[10], a[11], a[13], a[14] is not None, a[16] is not None)


@pytest.mark.parametrize("crop_box", [None, (64, 32, 448, 480)])
def test_refined_frame_launches_and_bounded_ring(host, monkeypatch, tmp_path, crop_box):
    from emoportraits_b200 import video

    w, pipe, seen = _inferer(monkeypatch, depth=2)
    s2w = __import__("test_refine_stream_cpu")._s2_wrapper()
    n = 11
    got = video.render_video(w, _pils(1, 300, "RGBA")[0], _pils(n), tmp_path / "o.mp4", inferer_s2=s2w, crop_box=crop_box, size=256)
    assert got == n and len(pipe.subs) == n and seen[-1]["refine"] is s2w.model_two and seen[-1]["mix"] and not seen[-1]["mix_old"]
    assert all(s["st"] is w.identity and "bg" not in s for s in pipe.subs)
    names = [c[0] for c in host]
    per = ["emo_u8_to_image"] + ["emo_resample_u8"] * (3 if crop_box else 2)
    assert names == per * n, names[:8]
    rs = [_shape(c) for c in host if c[0] == "emo_resample_u8"]
    k = 3 if crop_box else 2
    if crop_box:
        x0, y0, x1, y1 = crop_box
        assert rs[0] == (512, 512, 0, x0, y0, x1 - x0, y1 - y0, 512, 512, 0, True, True)   # crop, BICUBIC back to 512
    assert rs[k - 2] == (512, 512, 0, 0, 0, 512, 512, 256, 256, 1, True, True)              # LANCZOS to the panel, BGR
    assert rs[k - 1] == (256, 256, 0, 0, 0, 256, 256, 256, 256, 1, False, False)            # the driver panel: a copy
    # the ring: 2 rows per frame in flight, each reused only after its row was written out, rows written in order
    wr = _Writer.instances[-1]
    assert len(wr.rows) == n and wr.released and wr.args[2] == (768, 256)
    assert len({r.ctypes.data for r in wr.rows}) == 2 * pipe.depth
    rec = [e[1] for e in _Event.log if e[0] == "record"]
    sync = [e[1] for e in _Event.log if e[0] == "sync"]
    assert sync == rec                                                     # every row synchronised once, in order
    pos = {e: i for i, e in enumerate(_Event.log)}
    for i in range(2 * pipe.depth, n):
        assert pos[("sync", rec[i - 2 * pipe.depth])] < pos[("record", rec[i])]


def test_stage1_frames_from_a_video_path(host, monkeypatch, tmp_path):
    import cv2

    from emoportraits_b200 import video

    path = tmp_path / "d.mp4"
    frames = [np.full((90, 160, 3), i, np.uint8) for i in range(5)]

    class _Cap:
        def __init__(self, p):
            self.p, self.i = p, 0

        def isOpened(self):
            return self.p == str(path)

        def read(self):
            self.i += 1
            return (True, frames[self.i - 1]) if self.i <= len(frames) else (False, None)

        def release(self):
            pass

    monkeypatch.setattr(cv2, "VideoCapture", _Cap)
    w, pipe, seen = _inferer(monkeypatch)
    matte = []
    mask_fn = lambda x: matte.append(tuple(x.shape)) or torch.zeros(x.shape[0], 1, *x.shape[2:])   # noqa: E731
    monkeypatch.setattr(video, "STAGE1_CHUNK", 2)
    got = video.render_video(w, _pils(1)[0], str(path), tmp_path / "o.mp4", bg=torch.rand(3, 256, 256), mask_fn=mask_fn, size=128)
    assert got == 5 and len(_Writer.instances[-1].rows) == 5 and seen[-1]["refine"] is None
    assert matte == [(2, 3, 256, 256), (2, 3, 256, 256), (1, 3, 256, 256)]          # drive_image_with_video's batches
    assert all("dev_out" in s for s in pipe.subs)
    names = [c[0] for c in host]
    frame = ["emo_resample_u8", "emo_u8_to_image", "emo_resize_bicubic"]          # decode -> 128^2 RGB -> the model's 256^2
    assert names[:6] == frame * 2 and names[6:8] == ["emo_composite", "emo_image_to_u8"]
    assert names[8:12] == ["emo_resample_u8"] * 4
    rs = [_shape(c) for c in host if c[0] == "emo_resample_u8"]
    assert rs[0] == (90, 160, 1, 0, 0, 160, 90, 128, 128, 0, True, True)              # BGR decode, BICUBIC, to RGB
    assert rs[2] == (256, 256, 0, 0, 0, 256, 256, 128, 128, 1, True, True)            # output panel, LANCZOS, BGR
    assert rs[3] == (128, 128, 0, 0, 0, 128, 128, 128, 128, 1, False, False)          # driver panel: a copy


def test_refusals_queue_nothing(host, monkeypatch, tmp_path):
    from emoportraits_b200 import video

    w, pipe, seen = _inferer(monkeypatch)
    src, pils = _pils(1)[0], _pils(3)
    bg, mask_fn = torch.rand(3, 256, 256), (lambda x: x[:, :1])
    bad = [dict(frames=_pils(2, mode="RGBA")), dict(frames=_pils(2, mode="L")), dict(frames=pils, bg=bg),
           dict(frames=pils, mask_fn=mask_fn), dict(frames=pils, crop_box=(10, 10, 10, 50)),
           dict(frames=pils, crop_box=(10, 60, 50, 50)), dict(frames=pils, crop_box=(0.5, 0, 100, 100)),
           dict(frames=pils, crop_box=(0, 0, 100)),
           dict(frames=pils, inferer_s2=__import__("test_refine_stream_cpu")._s2_wrapper(), bg=torch.rand(3, 512, 512),
                mask_fn=mask_fn)]
    for kw in bad:
        with pytest.raises(ValueError):
            video.render_video(w, src, path=tmp_path / "o.mp4", **kw)
    with pytest.raises(FileNotFoundError):
        video.render_video(w, src, str(tmp_path / "missing.mp4"), tmp_path / "o.mp4")
    none, pipe_none, _ = _inferer(monkeypatch, state=False)
    with pytest.raises(RuntimeError, match="source"):
        video.render_video(none, src, pils, tmp_path / "o.mp4")
    assert not host and not pipe.subs and not pipe_none.subs and not _Writer.instances and not seen


@pytest.mark.parametrize("src_size", [512, 300])
def test_get_bg_launches(host, src_size):
    from emoportraits_b200 import video

    seen = {}

    def inpaint(gt, mask):
        seen["inpaint"] = (tuple(gt.shape), tuple(mask.shape))
        return torch.rand(1, 3, src_size, src_size)

    bg, bg_img = video.get_bg(_pils(1, src_size, "RGBA")[0], inpaint, lambda x: torch.rand(1, 1, *x.shape[2:]), 512, device="cpu")
    assert seen["inpaint"] == ((1, 3, src_size, src_size), (1, 1, src_size, src_size))
    assert tuple(bg.shape) == (3, 512, 512) and bg_img.size == (src_size, src_size) and bg_img.mode == "RGB"
    names = [c[0] for c in host]
    tail = ["emo_resample_u8", "emo_u8_to_image"] if src_size != 512 else ["emo_u8_to_image"]
    assert names == ["emo_u8_to_image", "emo_mask_dilate", "emo_image_to_u8"] + tail
    dil = host[1][1]
    assert dil[1:4] == (1, src_size, src_size) and dil[4].value == pytest.approx(0.8) and dil[5] == 20
