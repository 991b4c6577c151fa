"""The generation funnel on H100 — drop-in for the hot-path part of the reference's ``src/core.py``.

Kept verbatim from the reference: the generator contract of ``core_generation_funnel`` (src/core.py:83 — alias
``run_depthmap``, its historical name): ``(outpath, inputimages, inputdepthmaps, inputnames, inp, ops=None)`` ->
yields ``(input_index, kind, result)`` in the reference's order, with the same kinds and Python/PIL result types.
Every compute stage runs in the CUDA kernels of this package; images of equal size are processed as one batch
(the reference's strictly serial loop, src/core.py:133, is the thing being accelerated).

Out of the hot-path scope (SURVEY.md §8): background removal, heatmap, meshes, 3D inpainting.  Requesting them raises
``NotImplementedError`` naming the option instead of silently producing something else.
"""
from __future__ import annotations

import enum

import numpy as np
from PIL import Image

from . import _lib
from .normalmap_generation import create_normalmap_batch
from .stereoimage_generation import create_stereoimages_batch


class GenerationOptions(enum.Enum):
    """Option names + defaults consumed by the funnel (reference: src/common_constants.py:4-66)."""

    def __new__(cls, *args, **kwds):
        obj = object.__new__(cls)
        obj._value_ = len(cls.__members__) + 1
        return obj

    def __init__(self, default_value=None, *args):
        self.df = default_value

    COMPUTE_DEVICE = "GPU"
    MODEL_TYPE = "Depth Anything v2 Base"
    BOOST = False
    NET_SIZE_MATCH = False
    NET_WIDTH = 448
    NET_HEIGHT = 448
    TILING_MODE = False
    DO_OUTPUT_DEPTH = True
    OUTPUT_DEPTH_INVERT = False
    OUTPUT_DEPTH_COMBINE = False
    OUTPUT_DEPTH_COMBINE_AXIS = "Horizontal"
    DO_OUTPUT_DEPTH_PREDICTION = False
    CLIPDEPTH = False
    CLIPDEPTH_MODE = "Range"
    CLIPDEPTH_FAR = 0.0
    CLIPDEPTH_NEAR = 1.0
    GEN_STEREO = False
    STEREO_MODES = ["left-right", "red-cyan-anaglyph"]
    STEREO_DIVERGENCE = 2.5
    STEREO_SEPARATION = 0.0
    STEREO_FILL_ALGO = "polylines_sharp"
    STEREO_OFFSET_EXPONENT = 1.0
    STEREO_BALANCE = 0.0
    GEN_NORMALMAP = False
    NORMALMAP_PRE_BLUR = False
    NORMALMAP_PRE_BLUR_KERNEL = 3
    NORMALMAP_SOBEL = True
    NORMALMAP_SOBEL_KERNEL = 3
    NORMALMAP_POST_BLUR = False
    NORMALMAP_POST_BLUR_KERNEL = 3
    NORMALMAP_INVERT = False
    GEN_HEATMAP = False
    GEN_SIMPLE_MESH = False
    SIMPLE_MESH_OCCLUDE = True
    SIMPLE_MESH_SPHERICAL = False
    GEN_INPAINTED_MESH = False
    GEN_INPAINTED_MESH_DEMOS = False
    GEN_REMBG = False
    SAVE_BACKGROUND_REMOVAL_MASKS = False
    PRE_DEPTH_BACKGROUND_REMOVAL = False
    REMBG_MODEL = "u2net"


go = GenerationOptions

_OUT_OF_SCOPE = ("GEN_HEATMAP", "GEN_SIMPLE_MESH", "GEN_INPAINTED_MESH", "GEN_REMBG")


class CoreGenerationFunnelInp:
    """Case-insensitive option bag; unknown keys are silently dropped (reference: src/core.py:61-80)."""

    def __init__(self, values):
        if isinstance(values, CoreGenerationFunnelInp):
            values = values.values
        norm = {}
        for k, v in values.items():
            name = getattr(k, "name", k)
            norm[str(name).lower()] = v
        self.values = {}
        for setting in GenerationOptions:
            name = setting.name.lower()
            self.values[name] = norm[name] if name in norm else setting.df

    def __getitem__(self, item):
        name = getattr(item, "name", item)
        return self.values[str(name).lower()]

    def __getattr__(self, item):
        if item == "values":
            raise AttributeError(item)
        return self[item]


# ---------------------------------------------------------------------------------------------------------------------
# stage functions (batched, device in / device out)
# ---------------------------------------------------------------------------------------------------------------------
def percentile_plan(n, fractions):
    """Where np.percentile(a, [f*100 for f in fractions]) (method "linear", a.size == n) looks: for every fraction the two
    0-based ranks it reads and the float64 interpolation weight.  Same expressions, same order of operations as numpy's
    _QuantileMethods['linear'] / _get_indexes / _get_gamma (numpy/lib/_function_base_impl.py) so the weights are bit-identical."""
    q = np.true_divide(np.asanyarray([f * 100.0 for f in fractions], dtype=np.float64), np.float32(100))
    if not ((q >= 0).all() and (q <= 1).all()):
        raise ValueError("Percentiles must be in the range [0, 100]")       # numpy's own message
    virtual = (n - 1) * q                                  # _QuantileMethods["linear"]["get_virtual_index"]
    previous = np.floor(virtual).astype(np.intp)
    nxt = previous + 1
    above = virtual >= n - 1
    previous[above] = -1
    nxt[above] = -1
    below = virtual < 0
    previous[below] = 0
    nxt[below] = 0
    gamma = np.asanyarray(virtual - previous, dtype=virtual.dtype)
    return [(int(p) % n, int(x) % n, float(g)) for p, x, g in zip(previous, nxt, gamma)]


def normalize_prediction_batch(pred, invert=False, clipdepth=False, clipdepth_mode="Range", far=0.0, near=1.0,
                               return_flags=False):
    """Model prediction float32 CUDA [B,H,W] -> uint16 depth (near = bright).  src/core.py:189-211 + :44-50."""
    import ctypes
    import torch
    _lib.require_cuda()
    if pred.dtype != torch.float32:
        raise ValueError("prediction must be float32 (the reference's get_raw_prediction returns float32)")
    pred = pred.contiguous()
    B, H, W = pred.shape
    L = _lib.load()
    out = torch.empty((B, H, W), dtype=torch.uint16, device=pred.device)
    flags = torch.empty((B,), dtype=torch.int32, device=pred.device)
    if clipdepth and clipdepth_mode == "Outliers":      # src/core.py:200-202
        (p0, n0, g0), (p1, n1, g1) = percentile_plan(H * W, [far, near])
        ranks = (ctypes.c_int64 * 4)(p0, n0, p1, n1)
        ws_bytes = L.dm_normalize_u16_outliers_workspace_bytes(B)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=pred.device)
        rc = L.dm_normalize_u16_outliers(pred.data_ptr(), B, H, W, 1 if invert else 0, ranks, g0, g1, out.data_ptr(), flags.data_ptr(),
                                         ws.data_ptr(), ws_bytes, _lib.stream_ptr())
        _lib.check(rc, "dm_normalize_u16_outliers")
        return (out, flags) if return_flags else out
    # any other mode string: the reference has no else branch (src/core.py:197-202) and leaves the prediction unclipped
    mode = 1 if (clipdepth and clipdepth_mode == "Range") else 0
    ws_bytes = L.dm_normalize_u16_workspace_bytes(B)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=pred.device)
    rc = L.dm_normalize_u16(pred.data_ptr(), B, H, W, 1 if invert else 0, mode, float(far), float(near), out.data_ptr(),
                            flags.data_ptr(), ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "dm_normalize_u16")
    return (out, flags) if return_flags else out


def convert_to_i16(arr):
    """Single channel, 16 bit image from values in [0, 1) (reference: src/core.py:44-50); float32 in, uint16 out.

    For a model prediction use :func:`normalize_prediction_batch`, which fuses the min/max normalisation."""
    import torch
    dev = _lib.require_cuda()
    a = np.asarray(arr)
    if a.dtype == np.float64:
        return convert_to_i16_batch(torch.from_numpy(np.ascontiguousarray(a)).to(dev)).cpu().numpy()
    # float32 input: numpy keeps float32 arithmetic (Python scalars are weakly typed)
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    max_val = 2 ** 16
    out = torch.clamp(t * max_val + 0.0001, 0, max_val - 0.1)
    return out.to(torch.int32).cpu().numpy().astype("uint16")


def convert_to_i16_batch(t):
    """float64 CUDA tensor in [0, 1) -> uint16 CUDA tensor; the arithmetic of src/core.py:44-50 in float64 (what numpy
    does for the float64 custom depth maps of src/core.py:146-174) — dm_convert_to_i16_f64."""
    import torch
    t = t.to(torch.float64).contiguous()
    out = torch.empty(t.shape, dtype=torch.uint16, device=t.device)
    _lib.check(_lib.load().dm_convert_to_i16_f64(t.data_ptr(), t.numel(), out.data_ptr(), _lib.stream_ptr()), "dm_convert_to_i16_f64")
    return out


def convert_i16_to_rgb(image, like):
    """reference: src/core.py:52-58 (host-side formatting helper for OUTPUT_DEPTH_COMBINE)."""
    output = np.zeros_like(like)
    for k in range(3):
        output[:, :, k] = image / 256.0
    return output


# ---------------------------------------------------------------------------------------------------------------------
# the funnel
# ---------------------------------------------------------------------------------------------------------------------
_model_holder = None


def get_model_holder():
    global _model_holder
    if _model_holder is None:
        from .depthmap_generation import ModelHolder
        _model_holder = ModelHolder()
    return _model_holder


def _custom_depth_to_unit(dp, image):
    """reference: src/core.py:146-174 — host-side format handling of a user-supplied depth map."""
    if isinstance(dp, Image.Image):
        if dp.width != image.width or dp.height != image.height:
            try:
                dp = dp.resize((image.width, image.height), Image.Resampling.LANCZOS)
            except Exception:
                dp = dp.resize((image.width, image.height))
        if len(dp.getbands()) == 1:
            out = np.asarray(dp, dtype="float")
            out_max = out.max()
            bit_depth = 8 if out_max < 256 else (16 if out_max < 65536 else 32)
            out = out / 2.0 ** bit_depth
        else:
            out = np.asarray(dp, dtype="float")[:, :, 0] / 256.0
    else:
        out = np.asarray(dp, dtype="float")
        assert image.height == out.shape[0], "Custom depthmap height mismatch"
        assert image.width == out.shape[1], "Custom depthmap width mismatch"
    return out


def max_batch_for(width, height):
    """Upper bound on the images of one funnel batch (ADVICE r1: video mode hands every frame of a clip to one call).
    Bounded by pixel count so that the per-batch activation buffers stay at a few GB whatever the clip length;
    DEPTHMAP_B200_MAX_BATCH overrides."""
    import os
    env = os.environ.get("DEPTHMAP_B200_MAX_BATCH")
    if env:
        return max(1, int(env))
    return int(max(1, min(64, (1 << 24) // max(1, int(width) * int(height)))))


def _net_request(inp, w, h):
    """the (net_width, net_height) the funnel asks the model for on a w x h image"""
    if inp[go.NET_SIZE_MATCH]:
        return (w + 31) // 32 * 32, (h + 31) // 32 * 32
    return inp[go.NET_WIDTH], inp[go.NET_HEIGHT]


def _group_key(holder, inp, image, custom, boost):
    """Images with the same key form one device batch.  A depth-model image is keyed by its network input size (and the net size
    asked for), so images of different pixel sizes that share it run as one ragged forward; custom depth maps and BOOST (per image
    by design) keep the pixel size."""
    if custom or boost:
        return ("pixels", image.width, image.height, custom)
    req = _net_request(inp, image.width, image.height)
    return ("net", req, holder.net_size(image.width, image.height, *req))


def _process_chunk(holder, inp, dev, images, depthmaps, idxs, finish):
    """One batch of images with one group key through every requested stage on the device; returns `finish`'s per-image results.
    A batch of one pixel size runs as one uniform batch; a mixed one predicts as one ragged batch, then runs the later stages per
    run of equally sized images."""
    import torch
    rgbs = [np.asarray(images[i].convert('RGB') if images[i].mode != 'RGB' else images[i]) for i in idxs]
    if len({r.shape for r in rgbs}) == 1:
        return _process_run(holder, inp, dev, images, depthmaps, idxs, rgbs, None, finish)
    # one host -> device copy: the packed images
    layout = _lib.Ragged([r.shape[:2] for r in rgbs], 3, None)
    packed = torch.from_numpy(np.concatenate([r.reshape(-1) for r in rgbs])).to(dev, non_blocking=True)
    imgs = layout.split(packed)
    w0, h0 = images[idxs[0]].width, images[idxs[0]].height
    preds, invert = holder.get_raw_prediction_ragged(imgs, *_net_request(inp, w0, h0))
    out, j = [], 0
    while j < len(idxs):
        k = j + 1
        while k < len(idxs) and rgbs[k].shape == rgbs[j].shape:
            k += 1
        out += _process_run(holder, inp, dev, images, depthmaps, idxs[j:k], rgbs[j:k],
                            (torch.stack(imgs[j:k]), torch.stack(preds[j:k]), invert), finish)
        j = k
    return out


def _process_run(holder, inp, dev, images, depthmaps, idxs, rgbs, predicted, finish):
    """Equally sized images through every requested stage; `predicted` = (rgb batch, prediction batch, invert) when the depth model
    already ran on them.  `finish` turns the device results into per-image results (_HostImages or _PngFiles)."""
    import torch
    custom = depthmaps[idxs[0]] is not None
    preds = flags = None
    invert = False
    if predicted is not None:
        rgb_t, preds, invert = predicted
    else:
        rgb_t = torch.from_numpy(np.stack(rgbs)).to(dev, non_blocking=True)
    w, h = images[idxs[0]].width, images[idxs[0]].height
    if custom:
        outs = [_custom_depth_to_unit(depthmaps[i], images[i]) for i in idxs]
        depth_u16 = convert_to_i16_batch(torch.from_numpy(np.stack(outs)).to(dev))
    else:
        if preds is None:
            preds, invert = holder.get_raw_prediction_batch(rgb_t, *_net_request(inp, w, h))
        depth_u16, flags = normalize_prediction_batch(
            preds, invert, inp[go.CLIPDEPTH], inp[go.CLIPDEPTH_MODE], inp[go.CLIPDEPTH_FAR],
            inp[go.CLIPDEPTH_NEAR], return_flags=True)
    stereo = None
    if inp[go.GEN_STEREO]:
        stereo = create_stereoimages_batch(
            rgb_t, depth_u16, inp[go.STEREO_DIVERGENCE], inp[go.STEREO_SEPARATION], inp[go.STEREO_MODES],
            inp[go.STEREO_BALANCE], inp[go.STEREO_OFFSET_EXPONENT], inp[go.STEREO_FILL_ALGO])
    normal = None
    if inp[go.GEN_NORMALMAP]:
        normal = create_normalmap_batch(
            depth_u16,
            inp[go.NORMALMAP_PRE_BLUR_KERNEL] if inp[go.NORMALMAP_PRE_BLUR] else None,
            inp[go.NORMALMAP_SOBEL_KERNEL] if inp[go.NORMALMAP_SOBEL] else None,
            inp[go.NORMALMAP_POST_BLUR_KERNEL] if inp[go.NORMALMAP_POST_BLUR] else None,
            inp[go.NORMALMAP_INVERT])
    # the prediction crosses to the host only when it is yielded
    want_pred = preds is not None and inp[go.DO_OUTPUT_DEPTH_PREDICTION]
    preds_h = preds.cpu().numpy() if want_pred else None
    flags_h = flags.cpu().numpy() if want_pred else None
    pred_of = lambda j: None if preds_h is None else (preds_h[j], invert, int(flags_h[j]))
    return finish.run(inp, rgbs, rgb_t, depth_u16, pred_of, stereo, normal)


class _HostImages:
    """core_generation_funnel's results: one device -> host transfer per tensor per batch, PIL images made as they are yielded"""

    @staticmethod
    def run(inp, rgbs, rgb_t, depth_u16, pred_of, stereo, normal):
        depth_h = depth_u16.cpu().numpy()
        stereo_h = [s.cpu().numpy() for s in stereo] if stereo is not None else None
        normal_h = normal.cpu().numpy() if normal is not None else None
        return [(rgbs[j], depth_h[j], pred_of(j), None if stereo_h is None else [s[j] for s in stereo_h],
                 None if normal_h is None else normal_h[j]) for j in range(len(rgbs))]

    @staticmethod
    def depth(inp, rgb, img_output):
        img_depth = np.bitwise_not(img_output) if inp[go.OUTPUT_DEPTH_INVERT] else img_output
        if inp[go.OUTPUT_DEPTH_COMBINE]:
            axis = 1 if inp[go.OUTPUT_DEPTH_COMBINE_AXIS] == 'Horizontal' else 0
            return Image.fromarray(np.concatenate((rgb, convert_i16_to_rgb(img_depth, rgb)), axis=axis))
        return Image.fromarray(img_depth)

    @staticmethod
    def image(x):
        return Image.fromarray(x)


class _PngFiles:
    """core_generation_funnel_png's results: every image kind encoded to PNG on the device (invert and combine folded in), so only
    the compressed files cross to the host"""

    @staticmethod
    def run(inp, rgbs, rgb_t, depth_u16, pred_of, stereo, normal):
        from .png import combine_depth_rgb, encode_png_batch
        n = len(rgbs)
        depth = [None] * n
        if inp[go.DO_OUTPUT_DEPTH]:
            invert = bool(inp[go.OUTPUT_DEPTH_INVERT])
            if inp[go.OUTPUT_DEPTH_COMBINE]:
                horizontal = inp[go.OUTPUT_DEPTH_COMBINE_AXIS] == 'Horizontal'
                depth = encode_png_batch(combine_depth_rgb(rgb_t, depth_u16, horizontal, invert))
            else:
                depth = encode_png_batch(depth_u16, invert=invert)
        stereo_png = [encode_png_batch(s) for s in stereo] if stereo is not None else None
        normal_png = encode_png_batch(normal) if normal is not None else None
        return [(rgbs[j], depth[j], pred_of(j), None if stereo_png is None else [s[j] for s in stereo_png],
                 None if normal_png is None else normal_png[j]) for j in range(n)]

    @staticmethod
    def depth(inp, rgb, png):
        return png

    @staticmethod
    def image(png):
        return png


def core_generation_funnel(outpath, inputimages, inputdepthmaps, inputnames, inp, ops=None):
    return _funnel(outpath, inputimages, inputdepthmaps, inputnames, inp, ops, _HostImages)


def core_generation_funnel_png(outpath, inputimages, inputdepthmaps, inputnames, inp, ops=None):
    """core_generation_funnel with every image result as the bytes of a PNG file, encoded on the device (png.encode_png_batch):
    the same batching, options and (input_index, kind) sequence; `depth` (16-bit greyscale), `concat_depth`, every stereo mode and
    `normalmap` (8-bit RGB) are PNG bytes whose pixels equal the PIL image core_generation_funnel yields; `depth_prediction` is the
    same float array."""
    return _funnel(outpath, inputimages, inputdepthmaps, inputnames, inp, ops, _PngFiles)


def _funnel(outpath, inputimages, inputdepthmaps, inputnames, inp, ops, out_kind):
    if len(inputimages) == 0 or inputimages[0] is None:
        return
    if inputdepthmaps is None or len(inputdepthmaps) == 0:
        inputdepthmaps = [None for _ in range(len(inputimages))]
    inputdepthmaps_complete = all(x is not None for x in inputdepthmaps)
    inp = CoreGenerationFunnelInp(inp)
    for name in _OUT_OF_SCOPE:
        if inp[name]:
            raise NotImplementedError(f"{name} is outside the depthmap_b200 hot path (SURVEY.md §8); use the reference for it")
    holder = get_model_holder()
    if ops is None:
        ops = {}
    holder.update_settings(**ops)
    dev = _lib.require_cuda()  # COMPUTE_DEVICE == 'CPU' has no meaning here: there is no CPU path

    try:
        if not inputdepthmaps_complete:
            holder.ensure_models(inp[go.MODEL_TYPE], dev, inp[go.BOOST], inp[go.TILING_MODE])
        # single channel input (PIL mode I) -> RGB, as src/core.py:135-137 (the caller's list is updated, like the reference)
        for i in range(len(inputimages)):
            if inputimages[i].mode == 'I':
                inputimages[i] = inputimages[i].convert('RGB')

        # The reference loop is strictly serial (src/core.py:133).  Here consecutive images with one group key (_group_key:
        # the network input size for the depth model, so mixed pixel sizes can share a forward; the pixel size for custom depth
        # maps and BOOST) form one batch, bounded by max_batch_for of its largest image; batches are processed and yielded in
        # input order, so results stream out lazily and host / device memory stay bounded for long clips.
        modes = inp[go.STEREO_MODES]
        n = len(inputimages)
        boost = bool(inp[go.BOOST])
        key_of = lambda i: _group_key(holder, inp, inputimages[i], inputdepthmaps[i] is not None, boost)
        count = 0
        while count < n:
            key = key_of(count)
            idxs = [count]
            largest = inputimages[count].width * inputimages[count].height
            while idxs[-1] + 1 < n:
                nxt = inputimages[idxs[-1] + 1]
                grown = max(largest, nxt.width * nxt.height)
                if len(idxs) + 1 > max_batch_for(grown, 1) or key_of(idxs[-1] + 1) != key:
                    break
                idxs.append(idxs[-1] + 1)
                largest = grown
            results = _process_chunk(holder, inp, dev, inputimages, inputdepthmaps, idxs, out_kind)
            # yield in the reference's order (src/core.py:194-305)
            for i, (rgb, img_output, pred, stereo, normal) in zip(idxs, results):
                if pred is not None and inp[go.DO_OUTPUT_DEPTH_PREDICTION] and not pred[2]:
                    p = np.copy(pred[0])
                    if pred[1]:
                        p *= -1
                    yield i, 'depth_prediction', p
                if inp[go.DO_OUTPUT_DEPTH]:
                    yield i, 'concat_depth' if inp[go.OUTPUT_DEPTH_COMBINE] else 'depth', out_kind.depth(inp, rgb, img_output)
                if stereo is not None:
                    for c in range(len(stereo)):
                        yield i, modes[c], out_kind.image(stereo[c])
                if normal is not None:
                    yield i, 'normalmap', out_kind.image(normal)
            count = idxs[-1] + 1
    except Exception as e:
        if 'out of memory' in str(e).lower():
            # src/core.py:310-326: the reference replaces the error by its list of suggestions
            suggestion = "out of GPU memory, could not generate depthmap! Here are some suggestions to work around this issue:\n"
            if inp[go.BOOST]:
                suggestion += " * Disable BOOST (generation will be faster, but the depthmap will be less detailed)\n"
            suggestion += " * Use a different model (generally, more memory-consuming models produce better depthmaps)\n"
            if not inp[go.BOOST]:
                suggestion += " * Reduce net size (this could reduce quality)\n"
            suggestion += " * Lower DEPTHMAP_B200_MAX_BATCH (images per device batch)\n"
            raise Exception(suggestion)
        raise
    finally:
        if ops.get('depthmap_script_keepmodels', True):
            holder.offload()
        else:
            holder.unload_models()


run_depthmap = core_generation_funnel
