"""Mints tests/golden/*.npz by running the REAL reference (from /root/reference) in the build container.

    python tests/golden/make_golden.py

The GPU box has no /root/reference; tests there compare against these committed vectors (and against the oracle,
which tests/test_oracle_pin.py pins to the reference here).  Inputs are stored alongside outputs so the fixtures do
not depend on the synthetic generators staying unchanged.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.filterwarnings("ignore")

from oracle import ref_loader  # noqa: E402
from synth import noise_depth_u16, noise_rgb, synth_depth_u16, synth_rgb  # noqa: E402

FILLS = ['none', 'naive', 'naive_interpolating', 'polylines_soft', 'polylines_sharp']
STEREO_CASES = [  # (divergence, separation, balance, exponent)
    (2.5, 0.0, 0.0, 1.0), (5.0, 1.0, 0.3, 1.0), (10.0, -2.0, -0.5, 2.0), (0.05, 0.0, 0.0, 1.0), (15.0, 5.0, 1.0, 1.0),
    (4.0, 0.0, -1.0, 1.0),
]
NORMAL_CASES = [(None, 3, None, False), (None, 3, None, True), (None, 5, None, False), (None, 7, None, True),
                (None, None, None, False), (None, 1, None, False), (3, 3, None, False), (None, 3, 3, False),
                (5, 5, 5, True), (None, 9, None, False), (7, 3, 9, False)]


def main():
    ref = ref_loader.stereo_module()
    refn = ref_loader.normalmap_module()
    out = {}
    inputs = {
        "smooth": (synth_rgb(40, 56, 0), synth_depth_u16(40, 56, 0)),
        "noise": (noise_rgb(24, 64, 1), noise_depth_u16(24, 64, 1)),
    }
    blk = synth_rgb(32, 48, 2)
    blk[4:20, 8:30] = 0  # genuine black source pixels: exercises the sum()==0 logic of naive_interpolating
    inputs["black"] = (blk, synth_depth_u16(32, 48, 2))
    inputs["flat"] = (noise_rgb(8, 20, 3), np.full((8, 20), 1234, np.uint16))
    for name, (img, dep) in inputs.items():
        out[f"in_{name}_rgb"] = img
        out[f"in_{name}_depth"] = dep
        for fill in FILLS:
            for ci, (div, sep, bal, ex) in enumerate(STEREO_CASES):
                modes = ['left-right', 'red-cyan-anaglyph', 'top-bottom', 'cyan-red-reverseanaglyph']
                res = ref.create_stereoimages(img, dep, div, sep, modes, bal, ex, fill)
                for m, r in zip(modes, res):
                    out[f"stereo_{name}_{fill}_{ci}_{m}"] = np.asarray(r)
        if name != "flat":
            for ci, (pb, sb, qb, inv) in enumerate(NORMAL_CASES):
                out[f"normal_{name}_{ci}"] = np.asarray(refn.create_normalmap(dep, pb, sb, qb, inv))
    # split over four files of less than 1 MB each, largest arrays dealt first to the emptiest file
    parts, sizes = [{} for _ in range(4)], [0] * 4
    for k in sorted(out, key=lambda k: -np.asarray(out[k]).nbytes):
        i = sizes.index(min(sizes))
        parts[i][k] = out[k]
        sizes[i] += np.asarray(out[k]).nbytes
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(HERE, f"stereo_normal_golden_{i}.npz"), **part)
    print("wrote", len(out), "arrays")

    # funnel normalisation (src/core.py:189-211 + convert_to_i16) — executed through the reference's own functions
    import src.core as core  # noqa: E402  (module-level ModelHolder() only)
    rng = np.random.default_rng(7)
    nout = {}
    for i in range(6):
        raw = (rng.standard_normal((48, 64)) * 10 ** rng.uniform(-3, 3) + rng.uniform(-5, 5)).astype(np.float32)
        nout[f"pred_{i}"] = raw
        for inv in (False, True):
            for ci, (clip, far, near) in enumerate([(False, 0.0, 1.0), (True, 0.1, 0.8), (True, 0.0, 0.5)]):
                o = np.copy(raw)
                if inv:
                    o *= -1
                if clip:
                    o = (o - o.min()) / (o.max() - o.min())
                    o = np.clip(o, far, near)
                o = (o - o.min()) / (o.max() - o.min())
                nout[f"u16_{i}_{int(inv)}_{ci}"] = core.convert_to_i16(o)
    np.savez_compressed(os.path.join(HERE, "normalize_golden.npz"), **nout)
    print("wrote", len(nout), "arrays")


if __name__ == "__main__":
    main()
