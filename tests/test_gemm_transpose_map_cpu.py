"""The shared-memory transpose of pd_gemm_tf32_kernel (csrc/pd_gemm_sm90.cu, transpose_block), restated in numpy.

An MN-major operand tile lands from TMA in one of three forms: four 2-D boxes {32 mn, 32 k} 4096 B apart, one 3-D box
{32 mn, 32 k, 4 groups}, or (implicit convolution modes 2 and 3) four im2col boxes of 32 pixels (k) x 32 channels (mn).
wgmma reads tf32 operands only K-major, through a descriptor of a SWIZZLE_128B tile with row = mn and 32 k per 128-byte
row.  These tests check that the transposer warps' index map turns every landing form into exactly that tile, and that
none of its 16-byte shared-memory accesses has a bank conflict (each quarter-warp covers all 32 banks once)."""
import numpy as np
import pytest

TILE_WORDS = 128 * 32                  # one 16 KB fp32 operand tile


def swizzle128(byte):
    """TMA SWIZZLE_128B on a 1024-byte aligned tile: 16-byte chunk bits [4:6] XOR row bits [7:9]."""
    return byte ^ (((byte >> 7) & 7) << 4)


def land_mn_major(form):
    """word -> (mn, k) of a 128 x 32 MN-major tile as TMA lands it.  Every form writes boxes whose innermost dimension is
    32 mn (128 bytes) and whose rows are k; they differ in how the four 32-wide mn groups are addressed."""
    tile = np.full((TILE_WORDS, 2), -1, dtype=np.int64)
    for mn in range(128):
        for k in range(32):
            grp, c = mn // 32, mn % 32
            if form in ("2d", "im2col"):   # box j ({32 mn, 32 k}, or 32 pixels x 32 (tap, channel)) at j * 4096
                byte = grp * 4096 + swizzle128(k * 128 + c * 4)
            else:                          # one {32, 32, 4} box: 128 rows (group, k), swizzled as one tile
                byte = swizzle128((grp * 32 + k) * 128 + c * 4)
            tile[byte // 4] = (mn, k)
    assert (tile >= 0).all()
    return tile


def k_major_tile():
    """word -> (mn, k) of the K-major SWIZZLE_128B tile wg_desc describes: row = mn, chunk c of row r at c ^ (r & 7)."""
    tile = np.full((TILE_WORDS, 2), -1, dtype=np.int64)
    for mn in range(128):
        for k in range(32):
            byte = mn * 128 + (((k >> 2) ^ (mn & 7)) << 4) + (k & 3) * 4
            tile[byte // 4] = (mn, k)
    return tile


def swz(r, c):
    return r * 128 + ((c ^ (r & 7)) << 4)


def transpose_accesses(block):
    """The byte addresses of transpose_block on the 4 KB block `block` of a tile: per instruction, the 32 lanes'
    addresses.  Loads: (s, r) -> lane (q, p) reads k-row 4a + r at chunk p, a = p ^ (2q + s).  Stores: (s, i) -> lane
    writes mn-row 4p + i at chunk a the words (k = 4a + 0..3) it read from column i of its four loads."""
    base = block * 4096
    loads, stores = [], []
    for s in range(2):
        for r in range(4):
            loads.append([base + swz(4 * (p ^ (2 * (l >> 3) + s)) + r, p) for l in range(32) for p in [l & 7]])
    for s in range(2):
        for i in range(4):
            stores.append([base + swz(4 * p + i, p ^ (2 * (l >> 3) + s)) for l in range(32) for p in [l & 7]])
    return loads, stores


def run_transpose(tile):
    out = tile.copy()
    for block in range(4):
        loads, stores = transpose_accesses(block)
        regs = {}
        for n, addrs in enumerate(loads):            # n = 4 s + r
            for lane, a in enumerate(addrs):
                regs[(lane, n // 4, n % 4)] = [tile[a // 4 + w].copy() for w in range(4)]
        for n, addrs in enumerate(stores):           # n = 4 s + i
            s, i = n // 4, n % 4
            for lane, a in enumerate(addrs):
                for r in range(4):                   # word r of the store = element i of load r
                    out[a // 4 + r] = regs[(lane, s, r)][i]
    return out


@pytest.mark.parametrize("form", ["2d", "3d", "im2col"])
def test_transpose_yields_the_k_major_swizzled_tile(form):
    assert np.array_equal(run_transpose(land_mn_major(form)), k_major_tile())


def test_transpose_stays_inside_its_warps_4kb_block_and_covers_it_once():
    for block in range(4):
        loads, stores = transpose_accesses(block)
        for accesses in (loads, stores):
            words = sorted(a // 4 + w for addrs in accesses for a in addrs for w in range(4))
            assert words == list(range(block * 1024, (block + 1) * 1024))


def test_transpose_accesses_have_no_bank_conflicts():
    """A 16-byte access is served a quarter-warp (8 lanes) at a time; conflict-free when those 8 lanes hit 32 distinct
    banks."""
    for block in range(4):
        loads, stores = transpose_accesses(block)
        for addrs in loads + stores:
            assert all(a % 16 == 0 for a in addrs)
            for q in range(4):
                banks = {(a // 4 + w) % 32 for a in addrs[8 * q:8 * q + 8] for w in range(4)}
                assert len(banks) == 32
