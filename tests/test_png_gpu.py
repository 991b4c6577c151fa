"""GPU: PNG encoding on the device (dm_png_encode, png.encode_png_batch, core.core_generation_funnel_png).

  * lossless under two independent decoders (PIL, and OpenCV's libpng, which checks CRCs), uint16 and uint8 RGB, edge shapes;
  * stream structure: chunk CRCs, one IDAT per 32 KiB segment, the filtered stream (against a numpy restatement of the filter
    choice), Adler-32, and the size bound on noise;
  * a file depends on its image alone (batch, position, call);
  * core_generation_funnel_png yields what core_generation_funnel yields, as PNG files;
  * size against PIL's default save; errors."""
import io
import struct
import zlib

import numpy as np
import pytest
from PIL import Image

from synth import synth_depth_u16, synth_rgb

pytestmark = pytest.mark.gpu
SEG = 32768


def _enc(x, invert=False):
    import torch
    from depthmap_b200.png import encode_png_batch
    return encode_png_batch(torch.from_numpy(np.ascontiguousarray(x)).cuda(), invert=invert)


def _chunks(f):
    assert f[:8] == b"\x89PNG\r\n\x1a\n"
    out, p = [], 8
    while p < len(f):
        n, = struct.unpack(">I", f[p:p + 4])
        typ, data = f[p + 4:p + 8], f[p + 8:p + 8 + n]
        crc, = struct.unpack(">I", f[p + 8 + n:p + 12 + n])
        assert crc == zlib.crc32(typ + data), typ
        out.append((typ, data))
        p += 12 + n
    assert p == len(f) and out[-1] == (b"IEND", b"")
    return out


def _pil(f):
    im = Image.open(io.BytesIO(f))
    im.load()
    return im


def _cv2(f):
    import cv2
    return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_UNCHANGED)


def _raw_rows(x):
    """the unfiltered PNG scanlines of one image: 16-bit samples big-endian"""
    if x.dtype == np.uint16:
        return x.astype(">u2").view(np.uint8).reshape(x.shape[0], -1)
    return x.reshape(x.shape[0], -1)


def _filtered_ref(x):
    """PNG filtering with one filter per row by the minimum sum of absolute signed bytes (ties: the lower type)"""
    raw = _raw_rows(x).astype(np.int32)
    bpp = 2 if x.dtype == np.uint16 else 3
    H, R = raw.shape
    prev = np.zeros(R, np.int32)
    rows = []
    for y in range(H):
        r = raw[y]
        a = np.concatenate([np.zeros(bpp, np.int32), r])[:R]
        c = np.concatenate([np.zeros(bpp, np.int32), prev])[:R]
        b = prev
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        cands = [(v & 0xFF) for v in (r, r - a, r - b, r - ((a + b) >> 1), r - paeth)]
        f = int(np.argmin([int(np.where(v < 128, v, 256 - v).sum()) for v in cands]))
        rows.append(bytes([f]) + cands[f].astype(np.uint8).tobytes())
        prev = r
    return b"".join(rows)


def _check_file(f, x):
    """f decodes to x under both decoders, and its chunks are what the encoder promises"""
    pil = _pil(f)
    got = np.asarray(pil)
    assert got.dtype == x.dtype and got.shape == x.shape and np.array_equal(got, x)
    assert pil.mode == ("I;16" if x.dtype == np.uint16 else "RGB")
    cv = _cv2(f)
    want_cv = x if x.ndim == 2 else x[:, :, ::-1]
    assert cv is not None and cv.dtype == x.dtype and np.array_equal(cv, want_cv)
    ch = _chunks(f)
    assert ch[0][0] == b"IHDR" and all(t == b"IDAT" for t, _ in ch[1:-1])
    stream_len = x.shape[0] * (1 + _raw_rows(x).shape[1])
    idats = [d for t, d in ch if t == b"IDAT"]
    assert len(idats) == (stream_len + SEG - 1) // SEG + 1 and len(idats[-1]) == 4    # one IDAT per segment, then the Adler-32
    z = b"".join(idats)
    filtered = zlib.decompress(z)
    assert len(filtered) == stream_len
    assert struct.unpack(">I", idats[-1])[0] == zlib.adler32(filtered)
    for d in idats[1:-2]:                                                  # every segment but the last ends on the sync marker
        assert d.endswith(b"\x00\x00\xff\xff")
    return filtered


def _contents(h, w, rgb, seed):
    rng = np.random.default_rng(seed)
    shape = (h, w, 3) if rgb else (h, w)
    dt, top = (np.uint8, 256) if rgb else (np.uint16, 65536)
    yy, xx = np.mgrid[0:h, 0:w]
    grad = ((yy * 37 + xx * 91) * (top - 1) // max(1, (h - 1) * 37 + (w - 1) * 91)).astype(dt)
    row = rng.integers(0, top, (1,) + shape[1:], dtype=np.int64).astype(dt)
    return {
        "constant": np.full(shape, top // 3, dt),
        "gradient": np.repeat(grad[..., None], 3, axis=2) if rgb else grad,
        "repeated_rows": np.repeat(row, h, axis=0),
        "noise": rng.integers(0, top, shape, dtype=np.int64).astype(dt),
    }


SHAPES = [(1, 1), (1, 777), (513, 1), (37, 101), (64, 129)]


@pytest.mark.parametrize("rgb", [False, True], ids=["u16", "rgb8"])
@pytest.mark.parametrize("hw", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_lossless_and_structure(cuda_device, hw, rgb):
    h, w = hw
    for name, x in _contents(h, w, rgb, h * 1000 + w).items():
        f, = _enc(x[None])
        assert _check_file(f, x) == _filtered_ref(x), name


@pytest.mark.parametrize("rgb", [False, True], ids=["u16", "rgb8"])
def test_stream_ends_on_a_segment_boundary(cuda_device, rgb):
    h, w = (32768, 1) if not rgb else (4096, 5)            # 32768 rows of 3 bytes / 4096 rows of 16 bytes: exactly 3 and 2 segments
    assert h * (1 + w * (3 if rgb else 2)) % SEG == 0
    for name, x in _contents(h, w, rgb, 5).items():
        f, = _enc(x[None])
        assert _check_file(f, x) == _filtered_ref(x), name


@pytest.mark.parametrize("rgb", [False, True], ids=["u16", "rgb8"])
def test_4096_square(cuda_device, rgb):
    x = _contents(4096, 4096, rgb, 9)
    for name in ("gradient", "noise"):
        f, = _enc(x[name][None])
        _check_file(f, x[name])
    d = synth_depth_u16(4096, 4096, 3)
    if rgb:
        d = synth_rgb(4096, 4096, 3)
    f, = _enc(d[None])
    _check_file(f, d)


def test_bound_on_noise_and_entry_points(cuda_device):
    from depthmap_b200 import _lib
    L = _lib.load()
    for h, w, c, bits in ((300, 200, 1, 16), (300, 200, 3, 8), (1, 1, 1, 16), (4096, 5, 3, 8)):
        x = np.random.default_rng(h + w).integers(0, 1 << bits, (h, w) if c == 1 else (h, w, 3), dtype=np.int64)
        x = x.astype(np.uint16 if bits == 16 else np.uint8)
        f, = _enc(x[None])
        bound = L.dm_png_encode_bound(h, w, c, bits)
        stream = h * (1 + w * c * bits // 8)
        assert len(f) <= bound and bound == 63 + stream + 22 * ((stream + SEG - 1) // SEG)
        assert L.dm_png_encode_workspace_bytes(3, h, w, c, bits) > 3 * stream
    assert L.dm_png_encode_bound(4, 4, 3, 16) == 0 and L.dm_png_encode_workspace_bytes(1, 4, 4, 1, 8) == 0


def test_invert_flag(cuda_device):
    d = synth_depth_u16(90, 131, 4)
    f, = _enc(d[None], invert=True)
    _check_file(f, np.bitwise_not(d))


def test_depth_combine_rgb(cuda_device):
    import torch
    from depthmap_b200 import _lib
    from depthmap_b200.core import convert_i16_to_rgb
    from depthmap_b200.png import combine_depth_rgb
    rgb = np.stack([synth_rgb(41, 67, s) for s in range(3)])
    d = np.stack([synth_depth_u16(41, 67, s) for s in range(3)])
    for horizontal in (True, False):
        for invert in (False, True):
            got = combine_depth_rgb(torch.from_numpy(rgb).cuda(), torch.from_numpy(d).cuda(), horizontal, invert).cpu().numpy()
            for i in range(3):
                dd = np.bitwise_not(d[i]) if invert else d[i]
                want = np.concatenate((rgb[i], convert_i16_to_rgb(dd, rgb[i])), axis=1 if horizontal else 0)
                assert np.array_equal(got[i], want)
    # the C entry point directly
    out = torch.empty((1, 41, 134, 3), dtype=torch.uint8, device="cuda")
    r, dt = torch.from_numpy(rgb[:1]).cuda(), torch.from_numpy(d[:1]).cuda()
    _lib.check(_lib.load().dm_depth_combine_rgb(r.data_ptr(), dt.data_ptr(), 1, 41, 67, 1, 0, out.data_ptr(), _lib.stream_ptr()))
    assert np.array_equal(out[0].cpu().numpy()[:, 67:, 0], (d[0] >> 8).astype(np.uint8))


def test_file_depends_on_the_image_alone(cuda_device):
    rng = np.random.default_rng(11)
    imgs = [synth_depth_u16(120, 170, s) for s in range(8)]
    imgs[3] = rng.integers(0, 65536, (120, 170), dtype=np.int64).astype(np.uint16)
    imgs[5] = np.zeros((120, 170), np.uint16)
    alone = [_enc(x[None])[0] for x in imgs]
    batch = _enc(np.stack(imgs))
    assert batch == alone
    for pos in (0, 4, 7):                                  # the same image at several positions of a batch of 8
        order = [i for i in range(8) if i != 2]
        order.insert(pos, 2)
        got = _enc(np.stack([imgs[i] for i in order]))
        assert got[pos] == alone[2] and got == [alone[i] for i in order]
    assert _enc(np.stack(imgs)) == batch                   # a second call
    rgbs = np.stack([synth_rgb(77, 301, s) for s in range(8)])
    assert _enc(rgbs) == [_enc(x[None])[0] for x in rgbs]


def _pil_png_size(x):
    b = io.BytesIO()
    Image.fromarray(x).save(b, format="png")
    return len(b.getvalue())


def test_size_against_pil(cuda_device):
    """files of smooth depth maps and of funnel-like outputs are at most 1.3x the size of PIL's default PNG"""
    worst = 0.0
    for s, (h, w) in enumerate([(480, 640), (1080, 1920), (333, 517)]):
        d = synth_depth_u16(h, w, s)
        ratio = len(_enc(d[None])[0]) / _pil_png_size(d)
        worst = max(worst, ratio)
        print(f"depth {h}x{w}: {ratio:.3f}x PIL")
        assert ratio <= 1.3, (h, w, ratio)


ALL_MODES = ['left-right', 'right-left', 'top-bottom', 'bottom-top', 'red-cyan-anaglyph', 'left-only', 'only-right',
             'cyan-red-reverseanaglyph']


@pytest.fixture()
def funnel(cuda_device):
    from depthmap_b200 import core
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=2)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    yield core
    holder.unload_models()
    holder.weights_provider = None


def _opts(**kw):
    d = dict(compute_device='GPU', model_type=12, net_width=70, net_height=70, net_size_match=False, boost=False,
             do_output_depth=True, gen_stereo=False, gen_normalmap=False)
    d.update(kw)
    return d


def _same_as_plain(core, imgs, depthmaps, inp, ops=None, ratio=None):
    plain = list(core.core_generation_funnel(None, list(imgs), depthmaps, None, inp, ops=dict(ops or {})))
    png = list(core.core_generation_funnel_png(None, list(imgs), depthmaps, None, inp, ops=dict(ops or {})))
    assert [(i, k) for i, k, _ in png] == [(i, k) for i, k, _ in plain] and plain
    for (i, k, a), (_, _, b) in zip(plain, png):
        if k == 'depth_prediction':
            assert isinstance(b, np.ndarray) and np.array_equal(a, b)
            continue
        assert isinstance(b, bytes), k
        im = _pil(b)
        want = np.asarray(a)
        assert im.mode == ('I;16' if k == 'depth' else 'RGB') and a.mode in (('I;16',) if k == 'depth' else ('RGB',)), (k, im.mode, a.mode)
        assert np.array_equal(np.asarray(im), want), (i, k)
        cv = _cv2(b)
        assert np.array_equal(cv, want if want.ndim == 2 else want[:, :, ::-1]), (i, k)
        if ratio is not None and k in ('depth', 'normalmap'):
            ratio.append(len(b) / _pil_png_size(want))
    return plain, png


def test_funnel_png_all_outputs_mixed_sizes(funnel):
    core = funnel
    sizes = [(70, 98), (70, 98), (84, 70), (91, 123), (70, 98)]
    imgs = [Image.fromarray(synth_rgb(h, w, 30 + i)) for i, (h, w) in enumerate(sizes)]
    ratio = []
    _same_as_plain(core, imgs, None, _opts(gen_stereo=True, stereo_modes=ALL_MODES, gen_normalmap=True,
                                           do_output_depth_prediction=True), ratio=ratio)
    assert max(ratio) <= 1.3, ratio
    _same_as_plain(core, imgs, None, _opts(output_depth_invert=True, gen_normalmap=True, normalmap_invert=True))


@pytest.mark.parametrize("axis", ["Horizontal", "Vertical"])
@pytest.mark.parametrize("invert", [False, True])
def test_funnel_png_concat_depth(funnel, axis, invert):
    imgs = [Image.fromarray(synth_rgb(66, 90, s)) for s in range(3)]
    _same_as_plain(funnel, imgs, None, _opts(output_depth_combine=True, output_depth_combine_axis=axis, output_depth_invert=invert,
                                             gen_stereo=True, stereo_modes=['left-right']))


@pytest.mark.parametrize("mode", ["Range", "Outliers"])
def test_funnel_png_clip(funnel, mode):
    imgs = [Image.fromarray(synth_rgb(72, 96, s)) for s in range(2)]
    _same_as_plain(funnel, imgs, None, _opts(clipdepth=True, clipdepth_mode=mode, clipdepth_far=0.2, clipdepth_near=0.8,
                                             gen_normalmap=True, do_output_depth_prediction=True))


def test_funnel_png_custom_depthmaps(funnel):
    rgb = synth_rgb(40, 64, 7)
    d16 = synth_depth_u16(40, 64, 7)
    dm8 = Image.fromarray(np.repeat((d16 >> 8).astype(np.uint8)[:, :, None], 3, axis=2)).resize((32, 20))
    _same_as_plain(funnel, [Image.fromarray(rgb)] * 2, [Image.fromarray(d16), dm8],
                   _opts(gen_stereo=True, stereo_modes=['top-bottom', 'red-cyan-anaglyph'], gen_normalmap=True,
                         output_depth_combine=True, output_depth_combine_axis='Vertical'))
    _same_as_plain(funnel, [Image.fromarray(rgb)], [Image.fromarray(d16)], _opts(output_depth_invert=True))


def test_funnel_png_boost(cuda_device):
    from depthmap_b200 import core
    from oracle import synth_weights
    lsd = synth_weights.make_leres_state_dict(seed=2)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: psd if t == "pix2pix" else lsd
    try:
        img = Image.fromarray(synth_rgb(256, 320, 4))
        inp = dict(compute_device='GPU', model_type=0, net_width=448, net_height=448, boost=True, do_output_depth=True,
                   do_output_depth_prediction=True, gen_stereo=True, stereo_modes=['left-right'], gen_normalmap=True)
        plain, _ = _same_as_plain(core, [img], None, inp, ops={'boost_rmax': 1000})
        assert [k for _, k, _ in plain] == ['depth_prediction', 'depth', 'left-right', 'normalmap']
    finally:
        holder.unload_models()
        holder.weights_provider = None


def test_funnel_png_is_lazy(funnel):
    gen = funnel.core_generation_funnel_png(None, [Image.fromarray(synth_rgb(32, 32, 1))], None, None, _opts())
    assert next(gen)[1] == 'depth'


def test_errors(cuda_device):
    import torch
    from depthmap_b200 import _lib
    from depthmap_b200.png import combine_depth_rgb, encode_png_batch
    for bad in (torch.zeros((1, 4, 4), dtype=torch.float32, device="cuda"),
                torch.zeros((1, 4, 4), dtype=torch.uint8, device="cuda"),
                torch.zeros((1, 4, 4, 4), dtype=torch.uint8, device="cuda"),
                torch.zeros((4, 4), dtype=torch.uint16, device="cuda"),
                torch.zeros((1, 4, 4), dtype=torch.uint16),
                torch.zeros((0, 4, 4), dtype=torch.uint16, device="cuda"),
                np.zeros((1, 4, 4), np.uint16)):
        with pytest.raises(ValueError):
            encode_png_batch(bad)
    with pytest.raises(ValueError):
        encode_png_batch(torch.zeros((1, 4, 4, 3), dtype=torch.uint8, device="cuda"), invert=True)
    with pytest.raises(ValueError):
        combine_depth_rgb(torch.zeros((1, 4, 4, 3), dtype=torch.uint8, device="cuda"), torch.zeros((1, 4, 5), dtype=torch.uint16, device="cuda"))
    # short capacity / workspace: an error through _lib.check, and not one byte written
    L = _lib.load()
    B, H, W = 2, 50, 60
    x = torch.from_numpy(np.stack([synth_depth_u16(H, W, s) for s in range(B)])).cuda()
    bound = L.dm_png_encode_bound(H, W, 1, 16)
    ws_bytes = L.dm_png_encode_workspace_bytes(B, H, W, 1, 16)
    guard = 4096
    out = torch.full((B * bound + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    ws = torch.full((ws_bytes + guard,), 0x5A, dtype=torch.uint8, device="cuda")
    offsets = torch.full((B + 1,), -7, dtype=torch.int64, device="cuda")
    for cap, wsb in ((B * bound - 1, ws_bytes), (B * bound, ws_bytes - 1), (0, ws_bytes)):
        rc = L.dm_png_encode(x.data_ptr(), B, H, W, 1, 16, 0, out.data_ptr(), cap, offsets.data_ptr(), ws.data_ptr(), wsb,
                             _lib.stream_ptr())
        assert rc == _lib.DM_E_WORKSPACE
        with pytest.raises(RuntimeError, match="dm_png_encode"):
            _lib.check(rc, "dm_png_encode")
        torch.cuda.synchronize()
        assert bool((out == 0xA5).all()) and bool((ws == 0x5A).all()) and bool((offsets == -7).all())
    rc = L.dm_png_encode(x.data_ptr(), B, H, W, 1, 8, 0, out.data_ptr(), out.numel(), offsets.data_ptr(), ws.data_ptr(), ws_bytes,
                         _lib.stream_ptr())
    assert rc == _lib.DM_E_INVALID
    # exact capacity and workspace: the files fill [0, offsets[B]) and nothing past the capacity is touched
    rc = L.dm_png_encode(x.data_ptr(), B, H, W, 1, 16, 0, out.data_ptr(), B * bound, offsets.data_ptr(), ws.data_ptr(), ws_bytes,
                         _lib.stream_ptr())
    _lib.check(rc, "dm_png_encode")
    torch.cuda.synchronize()
    off = offsets.cpu().tolist()
    assert off[0] == 0 and off[-1] <= B * bound
    assert bool((out[B * bound:] == 0xA5).all()) and bool((ws[ws_bytes:] == 0x5A).all())
    data = out[:off[-1]].cpu().numpy().tobytes()
    for i in range(B):
        _check_file(data[off[i]:off[i + 1]], x[i].cpu().numpy())
