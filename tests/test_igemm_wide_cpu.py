"""b200_igemm_plan (host-only) for the convolutions of the C3 UNet (3-D, channels (256, 256, 512), 160 x 224 x 160) on a
132-SM H100: which calls take the 128 x 256 two-CTA kernel (column tile 256, work items = pairs of M tiles x column
tiles) and which stay on the 128-column kernel."""
import ctypes as C

from generativemodels_b200 import _lib


def plan(out_dhw, cout, segs, impl=0, n=1, stride=1, cols=None):
    """segs: number of filter-tap segments x 64-channel chunks per segment."""
    p = _lib.IgemmParams()
    p.in_N = p.out_N = n
    p.out_D, p.out_H, p.out_W = out_dhw
    p.in_D, p.in_H, p.in_W = (d * stride for d in out_dhw)
    p.stride_d = p.stride_h = p.stride_w = stride
    p.cout, p.out_cols = cout, cols or cout
    n_seg, nch = segs
    p.n_seg = n_seg
    for i in range(n_seg):
        p.seg[i].nchunks = nch
    p.impl = impl
    out = (C.c_int32 * 4)()
    assert _lib.load().b200_igemm_plan(C.byref(p), 132, 1, out) == 0
    return tuple(out)


L0, L1, L2 = (160, 224, 160), (80, 112, 80), (40, 56, 40)


def test_c3_convolutions_take_the_wide_kernel():
    # level 0, 27 taps x 4 chunks: 44 800 M tiles of 32 x 4 x 1 voxels -> 22 400 pairs
    assert plan(L0, 256, (27, 4)) == (256, 1, 22400, 0)
    # the concatenated 512 -> 256 conv1 of the up path: 27 taps x 2 sources x 4 chunks
    assert plan(L0, 256, (54, 4)) == (256, 1, 22400, 0)
    # level 1 (5 600 M tiles), its stride-2 downsample from level 0, and the 512-channel level 2 (700 M tiles x 2)
    assert plan(L1, 256, (27, 4)) == (256, 1, 2800, 0)
    assert plan(L1, 256, (27, 4), stride=2) == (256, 1, 2800, 0)
    assert plan(L2, 512, (27, 8)) == (256, 1, 700, 0)
    assert plan(L2, 512, (54, 8)) == (256, 1, 700, 0)


def test_upsample_phase_convolutions():
    # one output phase of the upsample into level 0: 8 taps x 4 chunks on the level-1 grid
    assert plan(L1, 256, (8, 4)) == (256, 1, 2800, 0)


def test_calls_that_keep_the_128_column_kernel():
    # GEMM-shaped calls (one segment), whatever their size
    assert plan((1, 1, 5734400), 256, (1, 108)) == (128, 1, 89600, 0)
    # too few units for one wave of 66 clusters: 8 x 8 x 16 voxels -> 8 M tiles
    assert plan((8, 8, 16), 256, (27, 4))[0] == 128
    # short reductions
    assert plan(L1, 256, (8, 2))[0] == 128
    # cout not a multiple of 256, or padded output columns
    assert plan(L1, 384, (27, 4))[0] == 128
    assert plan(L1, 256, (27, 4), cols=264)[0] == 128
    # impl 2 forces the 128-column kernel, impl 3 the wide one
    assert plan(L0, 256, (27, 4), impl=2) == (128, 1, 89600, 0)
    assert plan((8, 8, 16), 256, (27, 4), impl=3) == (256, 1, 4, 0)
    assert plan((1, 1, 1024), 256, (1, 4), impl=3)[0] == 256
