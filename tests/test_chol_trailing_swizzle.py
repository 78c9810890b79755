"""The shared-memory layout of the large Cholesky's trailing update (ba_chol_large.cu, chol_syrk_dmma_kernel): the pre-tiled
panel image is copied verbatim into shared memory, so its layout decides the bank pattern of the consumers' fragment loads.

This enumerates, for every consumer warp, every fragment load of every k8 step, which 16-byte bank group each lane hits, and
checks that the loads deliver exactly the m16n8k8 fragments of the plain row-major panel and are free of bank conflicts."""
import itertools

BT, BK = 128, 32               # SY_BT, SY_BK: one operand stage is 128 rows x 32 k
UNIT = 16                      # bytes per lane per fragment load (LDS.128)
GROUPS = 128 // UNIT           # 16-byte bank groups per 128-byte shared-memory wavefront


def img_index(r, k):
    """syrk_img_index inside one stage block: double offset of panel element (row r, k) for 0 <= r < 128, 0 <= k < 32"""
    t = k & 3
    u = 4 * t + ((k >> 3) ^ (t >> 1) ^ ((r & 1) << 1))
    return r * BK + 2 * u + ((k >> 2) & 1)


def consumer_offset(row, lane, s):
    """double offset of the 16-byte load a consumer lane issues for fragment row `row` (g, g + 8 plus a multiple of 8) in
    k8 step s: lane_a / lane_b + 2 (s ^ swz) in the kernel"""
    g, tg = lane >> 2, lane & 3
    swz = (tg >> 1) ^ ((g & 1) << 1)
    return row * BK + 8 * tg + 2 * (s ^ swz)


def fragment_rows(warp):
    """(row of lane group g = 0) of every 16-byte load of a consumer warp: A rows wr*64 + 16 i (+8), B rows wc*32 + 8 j"""
    wr, wc = warp >> 2, warp & 3
    a = [wr * 64 + 16 * i + h for i in range(4) for h in (0, 8)]
    b = [wc * 32 + 8 * j for j in range(4)]
    return a + b


def test_image_block_is_a_permutation_of_the_stage():
    offs = sorted(img_index(r, k) for r in range(BT) for k in range(BK))
    assert offs == list(range(BT * BK))


def test_each_load_returns_the_fragment_pair_t_and_t_plus_4():
    for warp, lane, s in itertools.product(range(8), range(32), range(4)):
        g, tg = lane >> 2, lane & 3
        for row0 in fragment_rows(warp):
            r = row0 + g
            off = consumer_offset(r, lane, s)
            assert off % 2 == 0                                  # 16-byte aligned
            assert img_index(r, 8 * s + tg) == off               # .x: k = 8 s + t
            assert img_index(r, 8 * s + tg + 4) == off + 1       # .y: k = 8 s + t + 4


def test_fragment_loads_are_free_of_bank_conflicts():
    """a 16-byte load of a warp is served as four quarter-warp wavefronts: the eight lanes of each must hit eight
    different bank groups (and, equivalently, every group is hit exactly four times by the whole warp)"""
    for warp, s in itertools.product(range(8), range(4)):
        for row0 in fragment_rows(warp):
            groups = [(consumer_offset(row0 + (lane >> 2), lane, s) * 8 // UNIT) % GROUPS for lane in range(32)]
            for q in range(4):
                assert len(set(groups[8 * q: 8 * q + 8])) == GROUPS, (warp, s, row0, groups)
            assert all(groups.count(x) == 4 for x in range(GROUPS))
