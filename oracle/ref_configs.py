"""Configurations for which the reference's kernel strings are compiled into oracle/_ref/ (TEST INFRASTRUCTURE).

The reference bakes (image_size, num_faces, texture_size, near, far, eps, return flags) into its CUDA source, so the
re-hosted reference needs one binary per configuration a test or the benchmark uses.  `cfg(...)` arguments are the
values the reference's `Rasterize.__init__` would receive (image_size is the RASTER size, i.e. already doubled for
anti-aliasing); near/far/eps keep their Python type because the reference pastes `str(value)` into the source.
"""
from build_ref import normalize_config as cfg

NEAR, FAR = 0.1, 100  # module defaults rasterize.py:9-10 (far is an int literal in the reference)
SIZES, SIZES_F, SIZES_TS = (255, 257, 700, 1024, 2048, 2051), 300, 2


def all_configs():
    c = []
    # known-answer gradient cases (tests/test_rasterize_silhouettes.py:37-99, tests/test_rasterize.py:76-149): fill_back -> F=2
    c.append(cfg(64, 2, 0, NEAR, FAR, 1e-4, 0, 1, 0))
    c.append(cfg(64, 2, 4, NEAR, FAR, 1e-3, 1, 0, 0))
    # teapot (2464 faces, fill_back -> 4928), Renderer paths: silhouette / depth use eps 1e-4, render uses 1e-3
    c.append(cfg(256, 4928, 0, NEAR, FAR, 1e-4, 0, 1, 0))
    c.append(cfg(256, 4928, 0, NEAR, FAR, 1e-4, 0, 0, 1))
    c.append(cfg(256, 4928, 4, NEAR, FAR, 1e-3, 1, 0, 0))
    c.append(cfg(512, 4928, 4, NEAR, FAR, 1e-3, 1, 0, 0))  # anti-aliased default Renderer (config 2 of BASELINE.json)
    c.append(cfg(128, 4928, 0, NEAR, FAR, 1e-4, 0, 1, 0))  # config 1: silhouette 64x64 with anti-aliasing
    # seeded random meshes
    c.append(cfg(32, 64, 2, NEAR, FAR, 1e-4, 1, 1, 1))
    for flags in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
        c.append(cfg(64, 200, 4 if flags[0] else 0, NEAR, FAR, 1e-4, *flags))
    c.append(cfg(100, 150, 3, NEAR, FAR, 1e-4, 1, 1, 1))   # raster size that is not a power of two
    c.append(cfg(128, 200, 4, NEAR, FAR, 1e-4, 1, 1, 1))   # used with anti_aliasing=True (image 64)
    c.append(cfg(64, 200, 2, 2.2, 3.0, 1e-4, 1, 1, 1))     # near / far rejection
    c.append(cfg(128, 24, 2, NEAR, FAR, 1e-4, 1, 1, 1))    # few large faces
    c.append(cfg(192, 2000, 2, NEAR, FAR, 1e-4, 1, 1, 0))  # 3x3 tiles, sphere mesh
    # headline shape (BASELINE.json metric): 256x256, 5000 faces
    c.append(cfg(256, 5000, 4, NEAR, FAR, 1e-4, 1, 0, 0))
    c.append(cfg(256, 5000, 2, NEAR, FAR, 1e-4, 1, 0, 0))
    c.append(cfg(256, 5000, 0, NEAR, FAR, 1e-4, 0, 1, 0))
    c.append(cfg(256, 5000, 0, NEAR, FAR, 1e-4, 0, 0, 1))
    # config 3 of BASELINE.json (bunny-scale): ~70k faces, depth + RGB, 512x512
    c.append(cfg(512, 70000, 2, NEAR, FAR, 1e-4, 1, 0, 1))
    # config 5 of BASELINE.json at reduced size: one shared 100k-face mesh, 512x512, RGB through Renderer.render (eps 1e-3)
    c.append(cfg(512, 100000, 2, NEAR, FAR, 1e-3, 1, 0, 0))
    # raster sizes that select other code paths of the product (tests/test_gpu_sizes.py, tests/test_gpu_uv.py): odd
    # sizes with a one-line last strip (255, 257), one-line strips (700, 1024), global-atomics binning (2048, 2051),
    # no pixel-centre table and a strip above 48 KB of shared memory (2051).  One (1, 1, 1) binary serves every
    # backward mode: the missing upstream gradients are zeros.
    for S in SIZES:
        c.append(cfg(S, SIZES_F, SIZES_TS, NEAR, FAR, 1e-4, 1, 1, 1))
    return c
