"""depthmap_b200 — H100-native drop-in for the depth -> 16-bit depth -> stereo / normal-map hot path of
thygate/stable-diffusion-webui-depthmap-script.

Public entry points keep the reference's names and signatures:

* ``stereoimage_generation.create_stereoimages``   (reference: src/stereoimage_generation.py:13)
* ``normalmap_generation.create_normalmap``         (reference: src/normalmap_generation.py:5)
* ``depthmap_generation.ModelHolder``               (reference: src/depthmap_generation.py:40)
* ``core.core_generation_funnel`` / ``core.run_depthmap`` / ``core.convert_to_i16``  (reference: src/core.py:83,44)

All compute runs in hand-written sm_90a CUDA kernels behind the C-ABI of ``include/depthmap_b200.h``
(``_native/libdepthmap_b200.so``, built by ``csrc/build.py``).  There is no CPU fallback: importing the operators
without the built library, or calling them without a CUDA device, raises.
"""
__version__ = "0.1.0"
