"""CPU model of the shared-memory layout of the experimental fused stem kernels (``csrc/kernels/stem_kernels.cu``).

The kernels cannot run here, but their index arithmetic can be checked: this test re-states, byte for byte, what
``load_patch`` + ``build_row`` write (zero-margined input rows → 16-byte chunks at swizzled positions of three
128-row x 128-byte k-blocks) and decodes the result with the CANONICAL wgmma layouts documented in CUTLASS
(``cute/atom/mma_traits_sm100.hpp``):

* K-major  SWIZZLE_128B: ``Swizzle<3,4,3> o ((8,m),(T,2)):((8T,SBO),(1,T))``          — the forward's A operand,
* MN-major SWIZZLE_128B: ``Swizzle<3,4,3> o ((T,8,m),(8,k)):((1,T,LBO),(8T,SBO))``    — the same bytes as the weight
  gradient's M-side operand (LBO = 16 KB between k-blocks, SBO = 1 KB between 8-pixel groups),

and compares against the patch matrix ``psb_im2col_stem`` defines (``ops/stem.py``: 7 kernel rows x 24 columns + 8 zeros).
"""
import numpy as np
import pytest

MARGIN = 48
SA_BLK = 128 * 128
T = 8                      # bf16 elements per 16 bytes


def swz(byte_off: int) -> int:
    """Swizzle<3,4,3> on a byte offset (tile base 1024-byte aligned): bits [4,7) ^= bits [7,10)."""
    return byte_off ^ (((byte_off >> 7) & 7) << 4)


def build_tile(x: np.ndarray, n: int, oh: int) -> np.ndarray:
    """Emulates load_patch + build_row for output row (n, oh).  x: [N,H,W,3] uint16 (bf16 bit patterns)."""
    _, H, W, _ = x.shape
    OW = (W - 1) // 2 + 1
    pitch = MARGIN + W * 6 + MARGIN
    patch = np.zeros(7 * pitch, dtype=np.uint8)
    for kh in range(7):                                     # load_patch: whole input rows, zero rows outside the image
        ih = 2 * oh - 3 + kh
        if 0 <= ih < H:
            patch[kh * pitch + MARGIN: kh * pitch + MARGIN + W * 6] = x[n, ih].reshape(-1).view(np.uint8)
    a = np.zeros(3 * SA_BLK, dtype=np.uint8)                # the A buffer was zeroed once
    for bt in range(OW):                                    # build_row, thread bt
        prow = 30 + 12 * bt
        arow = (bt >> 3) * 1024 + (bt & 7) * 128
        for kh in range(7):
            q = prow + kh * pitch
            src = patch[q: q + 48].copy()
            src[42:] = 0                                    # v[10] keeps element 20 only, v[11] = 0
            for c3 in range(3):
                qc = kh * 3 + c3
                dst = arow + (qc >> 3) * SA_BLK + (((qc & 7) ^ (bt & 7)) << 4)
                a[dst: dst + 16] = src[16 * c3: 16 * c3 + 16]
    return a


def im2col_row(x: np.ndarray, n: int, oh: int, ow: int) -> np.ndarray:
    """Row of the [N*OH*OW, 176] patch matrix as psb_im2col_stem writes it."""
    _, H, W, _ = x.shape
    row = np.zeros(176, dtype=np.uint16)
    for kh in range(7):
        ih = 2 * oh - 3 + kh
        if not 0 <= ih < H:
            continue
        for kw in range(7):
            iw = 2 * ow - 3 + kw
            if 0 <= iw < W:
                row[kh * 24 + kw * 3: kh * 24 + kw * 3 + 3] = x[n, ih, iw]
    return row


def read_k_major(a: np.ndarray, row: int, k: int) -> int:
    """Element (row, k) through the canonical K-major SW128 layout, k-blocks of 64 elements 16 KB apart."""
    blk, kk = divmod(k, 64)
    off = blk * SA_BLK + (row % 8) * (8 * T * 2) + (row // 8) * 1024 + kk * 2      # ((8,m),(T,2)):((8T,SBO),(1,T))
    p = blk * SA_BLK + swz(off - blk * SA_BLK)
    return int(a[p]) | int(a[p + 1]) << 8


def read_mn_major(a: np.ndarray, mn: int, kidx: int, lbo: int = SA_BLK, sbo: int = 1024) -> int:
    """Element (mn, kidx) through the canonical MN-major SW128 layout ((T,8,m),(8,k)):((1,T,LBO),(8T,SBO))."""
    mblk, r = divmod(mn, 64)
    off = (r % T) * 2 + (r // T) * (T * 2) + (kidx % 8) * (8 * T * 2) + (kidx // 8) * sbo
    p = mblk * lbo + swz(off)
    return int(a[p]) | int(a[p + 1]) << 8


@pytest.mark.parametrize("shape,n,oh", [((2, 16, 16, 3), 1, 0), ((2, 16, 16, 3), 0, 7), ((1, 30, 40, 3), 0, 5),
                                        ((1, 17, 8, 3), 0, 8), ((1, 12, 256, 3), 0, 3)])
def test_a_tile_matches_im2col_in_both_canonical_layouts(shape, n, oh):
    rng = np.random.default_rng(0)
    x = rng.integers(1, 65535, size=shape, dtype=np.uint16)
    W = shape[2]
    OW = (W - 1) // 2 + 1
    a = build_tile(x, n, oh)
    for ow in sorted({0, 1, OW // 2, OW - 2, OW - 1} & set(range(OW))):
        want = im2col_row(x, n, oh, ow)
        got_k = np.array([read_k_major(a, ow, k) for k in range(176)], dtype=np.uint16)
        assert np.array_equal(got_k, want), f"K-major view, ow={ow}"
        # weight gradient: the same bytes read as an MN-major operand (M = im2col column, K = pixel)
        got_mn = np.array([read_mn_major(a, k, ow) for k in range(176)], dtype=np.uint16)
        assert np.array_equal(got_mn, want), f"MN-major view, ow={ow}"
    # rows >= OW and columns 176..191 never receive data: they take part in MMAs and must read as zero
    for row in range(OW, 128, 17):
        assert all(read_k_major(a, row, k) == 0 for k in range(0, 192, 7))
    assert all(read_k_major(a, 0, k) == 0 for k in range(168, 192))


def test_staging_tile_swizzle_roundtrip():
    """Epilogue staging: lane == row writes chunk j at (j ^ (row & 7)) — what a SWIZZLE_128B TMA store expects, and
    what the BatchNorm column-sum loop reads back with ((ch >> 3) ^ (row & 7))."""
    tile = np.zeros(128 * 128, dtype=np.uint8)
    vals = np.arange(128 * 64, dtype=np.uint16).reshape(128, 64)
    for row in range(128):
        for j in range(8):
            dst = row * 128 + ((j ^ (row & 7)) << 4)
            tile[dst: dst + 16] = vals[row, 8 * j: 8 * j + 8].view(np.uint8)
    for row in (0, 5, 63, 111):
        for ch in (0, 7, 8, 31, 63):
            p = (ch & 7) * 2 + row * 128 + (((ch >> 3) ^ (row & 7)) << 4)
            assert (int(tile[p]) | int(tile[p + 1]) << 8) == vals[row, ch]
            assert p == swz(row * 128 + ch * 2)              # == the canonical 128B swizzle of the linear [row][64] tile
