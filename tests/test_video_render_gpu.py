"""The device-side video loop on the GPU: emo_resample_u8 / emo_mask_dilate, video.get_bg and video.render_video.

  * Resample: ops.resample_u8 equals the installed Pillow's Image.crop(box).resize(size, f) bit for bit on the grid of
    tests/test_video_render_cpu.py plus the shapes the video loop launches, for RGB and BGR sources and destinations, from a
    panel of a wider source into a panel of a wider row (the bytes around it untouched).
  * Dilation: ops.mask_dilate equals cv2.dilate((m >= thr), ones(21, 21), iterations=2) and scipy's maximum_filter(size=41,
    mode='constant'), with masks touching the borders.
  * Background: get_bg equals cell 40 computed the notebook's way (cv2.dilate on the host, ToPILImage, PIL BICUBIC) with the
    stand-in networks, bit for bit in the tensor and the PIL image, for a 512^2 source and a 300x260 one.
  * Rows: every row render_video hands to cv2.VideoWriter.write equals the row make_video hands to it for
    drive_image_with_video's outputs, stage 1 alone and refined, composited or not, with and without a crop box, from a list
    and from an mp4 path; and the mp4 it writes reads back with the frame count and size.
  * Launch coverage: every emo_resample_u8 / emo_mask_dilate launch of render_video and get_bg falls among the shapes and
    channel orders tested here."""
import gc

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import frames as FR
from test_refine_stream_gpu import _context, _wrapper
from test_video_render_cpu import FILTERS, RESAMPLE_CASES, pil_resample

pytestmark = pytest.mark.gpu

# the shapes render_video and get_bg launch in this file, on top of the CPU grid: (source h, w, box, (out w, h))
LOOP_CASES = [
    (512, 512, None, (256, 256)),                   # refined 512^2 frame -> 256^2 panel
    (512, 512, (64, 32, 448, 480), (512, 512)),     # the crop box of the rows test, back to 512^2
    (256, 256, None, (256, 256)),                   # a driver or stage-1 frame at the panel size: a copy
    (240, 320, None, (256, 256)),                   # a decoded frame of the test's mp4 -> the driver frame
    (300, 260, None, (512, 512)),                   # get_bg of a 300x260 source
]
GPU_CASES = RESAMPLE_CASES + LOOP_CASES
S = 256                      # panel size of the rows tests (stage 1 at 256^2, stage 2 at 512^2)
CROP = (64, 32, 448, 480)


@pytest.fixture(autouse=True)
def _release():
    """collect each test's wrappers and captured graphs here, with no capture in progress (tests/test_embedding_drive_gpu.py)"""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class StandInInpainter(nn.Module):
    """a seeded stand-in for the notebook's LaMa TorchScript (inpaint(img, mask) -> (1,3,H,W)): two small convolutions over the
    masked image and the mask, sigmoid output"""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(777)
        self.register_buffer("w1", torch.randn(8, 4, 3, 3, generator=g) * 0.3)
        self.register_buffer("w2", torch.randn(3, 8, 3, 3, generator=g) * 0.3)

    def forward(self, img, mask):
        x = torch.cat([img * (1 - mask), mask], 1)
        return torch.sigmoid(F.conv2d(torch.relu(F.conv2d(x, self.w1, padding=1)), self.w2, padding=1))


def _nets():
    from emoportraits_b200 import masks
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    return StubMODNet().cuda(), masks.FaceParsing(None, device="cuda", net=StubBiSeNet().cuda())


# ---- resample -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("filt", sorted(FILTERS))
@pytest.mark.parametrize("case", range(len(GPU_CASES)))
def test_resample_matches_pillow(filt, case):
    from emoportraits_b200 import ops

    H, W, box, (ow, oh) = GPU_CASES[case]
    a = np.random.default_rng(case).integers(0, 256, (H, W, 3), dtype=np.uint8)
    want = pil_resample(a, (ow, oh), filt, box)
    for src_bgr in (False, True):
        for dst_bgr in (False, True):
            wide = torch.randint(0, 256, (H, W + 7, 3), dtype=torch.uint8, device="cuda")       # the source: a panel of a wider image
            wide[:, 5:5 + W] = torch.from_numpy(a[:, :, ::-1].copy() if src_bgr else a).cuda()
            row = torch.full((oh, ow + 9, 3), 0xA5, dtype=torch.uint8, device="cuda")
            out = ops.resample_u8(wide[:, 5:5 + W], (ow, oh), filt, crop=box, dst=row[:, 4:4 + ow], src_bgr=src_bgr, dst_bgr=dst_bgr)
            got = out.cpu().numpy()
            assert np.array_equal(got[:, :, ::-1] if dst_bgr else got, want), (case, filt, src_bgr, dst_bgr)
            rest = torch.cat([row[:, :4].reshape(-1), row[:, 4 + ow:].reshape(-1)])
            assert bool((rest == 0xA5).all())


def test_resample_refuses_bad_arguments():
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    img = torch.zeros((10, 12, 3), dtype=torch.uint8, device="cuda")
    for crop in [(0, 0, 0, 5), (3, 0, 2, 5), (0.5, 0, 4, 4)]:
        with pytest.raises(ValueError):
            ops.resample_u8(img, (4, 4), "bicubic", crop=crop)
    with pytest.raises(ValueError):
        ops.resample_u8(img, (4, 4), "bilinear")
    t = ops.resample_taps(12, 4, "bicubic", "cuda")
    with pytest.raises(L.EmoError, match="taps"):       # taps for an axis whose size does not change
        L.call("emo_resample_u8", img.data_ptr(), 10, 12, 36, 0, 0, 0, 12, 10, img.data_ptr(), 10, 4, 36, 0, t.table.data_ptr(), t.kmax,
               t.table.data_ptr(), t.kmax, None, 0, 0, torch.cuda.current_stream().cuda_stream)


# ---- dilation -----------------------------------------------------------------------------------------------------------------
def _masks():
    g = torch.Generator().manual_seed(5)
    out = []
    for h, w in [(512, 512), (300, 260)]:
        m = torch.rand((1, 1, h, w), generator=g) * 0.79
        for y, x in [(0, 0), (h - 1, w // 2), (h // 3, w - 1), (h // 2, w // 2)]:   # corners and borders, and one inside
            m[0, 0, y, x] = 0.9
        m[0, 0, 7, 9] = 0.8                                                          # exactly at the threshold
        out.append(m)
    return out


def test_mask_dilate_matches_maximum_filter():
    from scipy.ndimage import maximum_filter

    from emoportraits_b200 import ops

    for m in _masks():
        got = ops.mask_dilate(m.cuda(), 0.8, 20).cpu().numpy()[0, 0]
        want = maximum_filter((m[0, 0] >= 0.8).float().numpy(), size=41, mode="constant")
        assert got.dtype == np.float32 and np.array_equal(got, want)


def test_mask_dilate_matches_cv2_dilate():
    cv2 = pytest.importorskip("cv2")
    from emoportraits_b200 import ops

    for m in _masks():
        got = ops.mask_dilate(m.cuda(), 0.8, 20).cpu().numpy()[0, 0]
        want = cv2.dilate((m >= 0.8).float()[0].permute(1, 2, 0).numpy(), np.ones((21, 21), "uint8"), iterations=2)
        assert np.array_equal(got, want)


# ---- background ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(512, 512), (300, 260)])
def test_get_bg_matches_the_notebook(hw):
    cv2 = pytest.importorskip("cv2")
    TF = pytest.importorskip("torchvision.transforms.functional")
    from PIL import Image

    from emoportraits_b200 import masks, video

    source = Image.fromarray(FR.smooth_array(512, 44)[:hw[0], :hw[1]]).convert("RGBA")
    modnet, face_idt = _nets()
    mask_fn, lama = masks.face_matte(face_idt, modnet), StandInInpainter().cuda()
    bg, bg_img = video.get_bg(source, lama, mask_fn, 512)
    # cell 40
    gt = TF.to_tensor(source)[:3].unsqueeze(0).cuda()
    m = mask_fn(gt)
    mask = (m >= 0.8).float()[0].permute(1, 2, 0)
    d = torch.FloatTensor(cv2.dilate(mask.cpu().numpy(), np.ones((21, 21), "uint8"), iterations=2)).unsqueeze(0).unsqueeze(0).cuda()
    want_img = TF.to_pil_image(lama(gt, d)[0])
    want = TF.to_tensor(want_img.resize((512, 512), Image.BICUBIC))
    assert np.array_equal(np.asarray(bg_img), np.asarray(want_img)) and bg_img.size == (hw[1], hw[0])
    assert bg.shape == (3, 512, 512) and bg.is_cuda and torch.equal(bg.cpu(), want)


# ---- rows ---------------------------------------------------------------------------------------------------------------------
class _Recorder:
    """cv2.VideoWriter stand-in that keeps a copy of every row"""
    rows = None

    def __init__(self, *a):
        _Recorder.rows = []

    def write(self, row):
        _Recorder.rows.append(np.array(row))

    def release(self):
        pass


def _mp4(path, n=5):
    import cv2

    wr = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), 30.0, (320, 240))
    for i in range(n):
        wr.write(np.ascontiguousarray(FR.smooth_array(320, 70 + i)[:240, :, ::-1]))
    wr.release()
    return path


@pytest.fixture(scope="module")
def ctx():
    return _context(256)


@pytest.fixture(scope="module")
def s2_root(tmp_path_factory):
    return tmp_path_factory.mktemp("s2v")


def _s2(root):
    from test_composite_refine_gpu import _s2_wrapper_at

    s2w = _s2_wrapper_at(root, 512)
    s2w.modnet, s2w.face_idt = _nets()
    return s2w


@pytest.mark.parametrize("refined,composited,crop,from_path", [
    (False, False, False, False), (False, True, True, True), (False, True, False, False),
    (True, True, True, False), (True, False, False, True), (True, False, True, False)])
def test_rows_match_make_video(ctx, s2_root, tmp_path, monkeypatch, refined, composited, crop, from_path):
    import cv2
    from PIL import Image

    from emoportraits_b200 import masks, video

    w = _wrapper(ctx)
    s2w = _s2(s2_root) if refined else None
    kw = dict(bg=FR.frame(256, 96, "smooth")[0].cuda(), mask_fn=masks.face_matte(*_nets()[::-1])) if composited else {}
    box = CROP if crop else None
    src = Image.fromarray(FR.smooth_array(320, 41)[:300, :300]).convert("RGBA")    # any mode and size: make_video's panel
    frames = str(_mp4(tmp_path / "d.mp4")) if from_path else [FR.pil(256, 50 + i, "smooth") for i in range(5)]
    monkeypatch.setattr(cv2, "VideoWriter", _Recorder)
    pils = video.get_video_frames_as_images(frames, S) if from_path else frames
    outs, crops, _ = video.drive_image_with_video(w, src, pils, s2w, crop_box=box, in_flight=refined, **kw)
    video.make_video(src, pils, crops if crop else outs, tmp_path / "a.mp4", size=S)
    want = _Recorder.rows
    n = video.render_video(w, src, frames, tmp_path / "b.mp4", s2w, crop_box=box, size=S, **kw)
    got = _Recorder.rows
    assert n == len(got) == len(want) == 5
    for i, (g, wnt) in enumerate(zip(got, want)):
        assert g.shape == (S, 3 * S, 3) and np.array_equal(g, wnt), (i, np.argwhere(g != wnt)[:3].tolist())


def test_render_video_writes_an_mp4(ctx, tmp_path):
    import cv2

    from emoportraits_b200 import video

    w = _wrapper(ctx)
    w.forward(FR.pil(256, 41, "smooth"), None, crop=False)
    n = video.render_video(w, FR.pil(256, 41, "smooth"), str(_mp4(tmp_path / "d.mp4", 7)), tmp_path / "o.mp4", size=S)
    cap = cv2.VideoCapture(str(tmp_path / "o.mp4"))
    shapes = []
    while True:
        ret, f = cap.read()
        if not ret:
            break
        shapes.append(f.shape)
    cap.release()
    assert n == 7 and shapes == [(S, 3 * S, 3)] * 7


# ---- launch coverage ----------------------------------------------------------------------------------------------------------
def test_launches_fall_in_tested_shapes(ctx, s2_root, tmp_path, monkeypatch):
    import cv2
    from PIL import Image

    from emoportraits_b200 import lib as L
    from emoportraits_b200 import masks, video

    seen = []
    record = L.call

    def call(name, *args):
        if name in ("emo_resample_u8", "emo_mask_dilate"):
            seen.append((name, args))
        return record(name, *args)

    mp4 = str(_mp4(tmp_path / "d.mp4"))
    monkeypatch.setattr(L, "call", call)
    monkeypatch.setattr(cv2, "VideoWriter", _Recorder)
    w = _wrapper(ctx)
    w.forward(FR.pil(256, 41, "smooth"), None, crop=False)
    mask_fn = masks.face_matte(*_nets()[::-1])
    for src in (FR.pil(512, 44, "smooth"), Image.fromarray(FR.smooth_array(512, 44)[:300, :260])):
        video.get_bg(src, StandInInpainter().cuda(), mask_fn, 512)
    bg = FR.frame(256, 96, "smooth")[0].cuda()
    video.render_video(w, FR.pil(256, 41, "smooth"), mp4, tmp_path / "o.mp4", _s2(s2_root), bg=bg,
                       mask_fn=mask_fn, crop_box=CROP, size=S)
    video.render_video(w, FR.pil(256, 41, "smooth"), [FR.pil(256, 50, "smooth")], tmp_path / "o.mp4", size=S)
    tested = {(H, W, box or (0, 0, W, H), size) for H, W, box, size in GPU_CASES}
    assert {n for n, _ in seen} == {"emo_resample_u8", "emo_mask_dilate"}
    for name, a in seen:
        if name == "emo_mask_dilate":
            assert (a[2], a[3], a[5]) in {(512, 512, 20), (300, 260, 20)} and a[1] == 1, a[:6]
            continue
        H, W, x0, y0, cw, ch, oh, ow = a[1], a[2], a[5], a[6], a[7], a[8], a[10], a[11]
        assert (H, W, (x0, y0, x0 + cw, y0 + ch), (ow, oh)) in tested, (H, W, x0, y0, cw, ch, ow, oh)
