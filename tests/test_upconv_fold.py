"""CPU tests of the sub-pixel form of `nearest x2 -> 3x3 conv` (emo_conv_desc.upconv, ops.fold_upconv_weight):
the weight folding is exact algebra, and the index arithmetic the CUDA kernel uses (conv_igemm.cu, conv_igemm_kernel with
PS = true: tile origin - pad + phase shift + tap, weight row phase * 4 + tap, output pixel 2 g + parity) is restated here
with torch gathers and compared with F.conv2d on the upsampled map."""
import torch
import torch.nn.functional as F


def _ref(x, w):
    return F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1)


def test_fold_matches_conv_on_upsampled_map():
    from emoportraits_b200.ops import fold_upconv_weight

    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 7, 9, generator=g)
    w = torch.randn(4, 5, 3, 3, generator=g)
    fw = fold_upconv_weight(w)                                        # (4 phases, 2, 2, Co, Ci)
    ref = _ref(x, w)
    out = torch.zeros_like(ref)
    for ph in range(4):
        pa, pb = ph >> 1, ph & 1
        k = fw[ph].permute(2, 3, 0, 1)                                # (Co, Ci, 2, 2)
        # parity 0 reads offsets {-1, 0}: pad one row/column before; parity 1 reads {0, +1}: pad one after
        xp = F.pad(x, (1 - pb, pb, 1 - pa, pa))
        out[:, :, pa::2, pb::2] = F.conv2d(xp, k)
    assert (out - ref).abs().max().item() < 1e-4 * ref.abs().max().item()


def test_kernel_index_arithmetic():
    """the integer formulas of the kernel, one 'tile' covering the whole low-res grid"""
    from emoportraits_b200.ops import fold_upconv_weight

    g = torch.Generator().manual_seed(1)
    N, Ci, Co, H, W = 1, 6, 4, 5, 8
    x = torch.randn(N, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g)
    wk = fold_upconv_weight(w).reshape(16, Co, Ci)                    # weight rows as the tensor map sees them
    ref = _ref(x, w)
    out = torch.full_like(ref, float("nan"))
    ph_pad, pw_pad, kh, kw = 1, 1, 2, 2                               # p.ph, p.pw of the descriptor; p.kh = p.kw = 2
    xcl = x.permute(0, 2, 3, 1)                                       # channels-last, as the TMA box reads it
    for ph in range(4):                                               # nt / p.ntc
        xs, ys = (1 if (ph & 1) else 0), (1 if (ph >> 1) else 0)
        acc = torch.zeros(N, H, W, Co)
        for tap in range(kh * kw):
            c, b = tap % kw + xs, (tap // kw) % kh + ys
            wtap = ph * 4 + tap
            for gh in range(H):
                for gw in range(W):
                    yy, xx = gh - ph_pad + b, gw - pw_pad + c         # y0 + b, x0 + c with tile origin (gh, gw)
                    if 0 <= yy < H and 0 <= xx < W:                   # TMA zero fill outside
                        acc[:, gh, gw] += xcl[:, yy, xx] @ wk[wtap].T
        for gh in range(H):
            for gw in range(W):
                out[:, :, 2 * gh + (ph >> 1), 2 * gw + (ph & 1)] = acc[:, gh, gw]
    assert not torch.isnan(out).any()
    assert (out - ref).abs().max().item() < 1e-4


def test_poolconv_fold_matches_conv_then_avgpool():
    """ops.fold_poolconv_weight: avgpool2(conv3x3(x, pad 1) + bias) == conv4x4(x, stride 2, pad 1) + bias"""
    from emoportraits_b200.ops import fold_poolconv_weight

    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 6, 10, 14, generator=g)
    w = torch.randn(5, 6, 3, 3, generator=g)
    b = torch.randn(5, generator=g)
    ref = F.avg_pool2d(F.conv2d(x, w, b, padding=1), 2)
    out = F.conv2d(x, fold_poolconv_weight(w), b, stride=2, padding=1)
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())


def _pick_box(dim, want):
    b = want
    while b > dim:
        b >>= 1
    return max(b, 1)


def test_subpixel_tile_walk_restated():
    """Host parameters (emo_conv_igemm, upconv branch) and device index logic (conv_igemm_kernel with PS = true)
    restated for a multi-tile case: 128-pixel boxes over the low-res grid, N tile = (phase, channel tile), TMA box gather
    with zero fill, pixel-shuffle store.  Every output element must be written exactly once with the reference value."""
    from emoportraits_b200.ops import fold_upconv_weight

    g = torch.Generator().manual_seed(3)
    N, Ci, Co, H, W = 2, 8, 64, 16, 32          # low-res grid 16 x 32 -> output 32 x 64
    x = torch.randn(N, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g)
    ref = _ref(x, w).permute(0, 2, 3, 1).contiguous()               # channels-last (N, 2H, 2W, Co)
    wk = fold_upconv_weight(w).reshape(16, Co, Ci)
    xcl = x.permute(0, 2, 3, 1).contiguous()
    # ---- host (emo_conv_igemm with d->upconv) ----
    BN = 32                                                          # a pair-compatible N tile dividing Cout_pad
    gH, gW, oH, oW = H, W, 2 * H, 2 * W
    tw = _pick_box(gW, 16); th = _pick_box(gH, 128 // tw); td = 1
    tiles_w, tiles_h, tiles_d = -(-gW // tw), -(-gH // th), 1
    m_tiles = N * tiles_d * tiles_h * tiles_w
    ntc = Co // BN
    n_tiles = 4 * ntc
    kh = kw = 2; ph_pad = pw_pad = 1
    assert m_tiles % 2 == 0                                          # pair mode
    out = torch.full((N, oH, oW, Co), float("nan"))
    writes = torch.zeros((N, oH, oW, Co), dtype=torch.int32)
    rows_a = tw * th * td
    for tile in range(m_tiles * n_tiles):
        nt = tile // m_tiles
        mt = tile - nt * m_tiles
        twi = mt % tiles_w; mt //= tiles_w
        thi = mt % tiles_h; mt //= tiles_h
        n = mt
        # ---- producer ----
        x0, y0 = twi * tw - pw_pad, thi * th - ph_pad
        ph = nt // ntc
        n0 = (nt - ph * ntc) * BN
        xs, ys = (1 if ph & 1 else 0), (1 if ph >> 1 else 0)
        acc = torch.zeros(rows_a, BN)
        for tap in range(kh * kw):
            c, b = tap % kw + xs, (tap // kw) % kh + ys
            wtap = ph * 4 + tap
            A = torch.zeros(rows_a, Ci)                               # TMA box {Ci, tw, th} at (x0 + c, y0 + b), zero fill
            for r in range(rows_a):
                xx, yy = x0 + c + r % tw, y0 + b + r // tw
                if 0 <= xx < W and 0 <= yy < H:
                    A[r] = xcl[n, yy, xx]
            acc += A @ wk[wtap, n0:n0 + BN].T
        # ---- accumulate / store role ----
        for row in range(rows_a):
            gw, gh = twi * tw + row % tw, thi * th + (row // tw) % th
            if gw < gW and gh < gH:
                ow, oh = 2 * gw + (ph & 1), 2 * gh + (ph >> 1)
                out[n, oh, ow, n0:n0 + BN] = acc[row]
                writes[n, oh, ow, n0:n0 + BN] += 1
    assert int(writes.min()) == 1 and int(writes.max()) == 1
    assert (out - ref).abs().max().item() < 1e-4
