"""Host-side emulation of index formulas used inside the CUDA kernels (no GPU needed), in the spirit of
tests/test_fft_indexing.py: each check restates a formula from the cited kernel source in numpy and proves the
property the kernel relies on (bijectivity, exact cover, balanced barrier traffic).  They guard the algebra, not the
CUDA text: when a formula in the kernel changes, the restatement here has to change with it."""
import numpy as np
import pytest


# ---- gemm_epilogue.cuh: epi_store_staged (swizzled smem staging, cooperative coalesced stores) ----------------
@pytest.mark.parametrize("out_bf16", [False, True])
def test_epilogue_staging_swizzle_is_a_bijection_and_stores_are_coalesced(out_bf16):
    row_bytes = 64 if out_bf16 else 128                     # 32 columns per chunk
    nseg = row_bytes // 16                                  # 16-byte segments per row
    buf = -np.ones((128 * row_bytes // 16,), dtype=np.int64)  # segment slot -> (row, logical segment)
    for r in range(128):                                    # writer: thread r owns row r
        sw = ((r >> 1) & 3) if out_bf16 else (r & 7)
        for j in range(nseg):
            slot = r * nseg + (j ^ sw)
            assert buf[slot] == -1                          # no two writes collide
            buf[slot] = r * 100 + j
    assert (buf >= 0).all()
    seen = set()
    for et in range(128):                                   # reader: cooperative pattern
        q = et & (nseg - 1)
        for i in range(nseg):
            row = i * (128 // nseg) + (et >> (2 if out_bf16 else 3))
            sw = ((row >> 1) & 3) if out_bf16 else (row & 7)
            v = buf[row * nseg + (q ^ sw)]
            assert v == row * 100 + q                       # reads back logical segment q of that row
            seen.add((row, q))
    assert len(seen) == 128 * nseg                          # every (row, segment) stored exactly once
    # coalescing: the nseg lanes with consecutive `et` cover one row contiguously
    for et0 in range(0, 128, nseg):
        rows = {(et >> (2 if out_bf16 else 3)) for et in range(et0, et0 + nseg)}
        assert len(rows) == 1


def test_single_cta_epilogue_groups_split_the_tile_in_halves():
    bn, groups = 128, 2                                     # GemmEpi<128>
    cols = [list(range(g * (bn // groups), (g + 1) * (bn // groups))) for g in range(groups)]
    assert sorted(sum(cols, [])) == list(range(bn))
    # consumer warpgroups 1-2 (threads 128..383) are the two groups; thread & 127 is the tile row in both
    for g in range(groups):
        threads = range(128 * (g + 1), 128 * (g + 2))
        assert {(t >> 7) - 1 for t in threads} == {g}
        assert sorted(t & 127 for t in threads) == list(range(128))


# ---- gemm_sm90.cuh: wgmma accumulator fragments -> the shared-memory accumulator tile ------------------------------
@pytest.mark.parametrize("bn", [64, 128])
def test_accumulator_fragments_fill_the_shared_tile_exactly_once(bn):
    cover = np.zeros((128, bn), dtype=int)
    for t in range(128, 384):                               # consumer threads
        wg, warp, lane = (t >> 7) - 1, (t >> 5) & 3, t & 31
        r = wg * 64 + warp * 16 + (lane >> 2)
        c = 2 * (lane & 3)
        for j in range(bn // 8):                            # acc[4j], acc[4j+1] -> row r; acc[4j+2], acc[4j+3] -> row r+8
            for rr in (r, r + 8):
                cover[rr, 8 * j + c:8 * j + c + 2] += 1
    assert (cover == 1).all()


# ---- gemm_sm90.cuh: weight tiles requested before the PDL wait --------------------------------------------------
@pytest.mark.parametrize("num_kb,stages", [(16, 6), (32, 6), (2, 6), (16, 3), (1, 4)])
def test_early_weight_tiles_plus_main_loop_issue_every_k_block_once(num_kb, stages):
    early_b = min(stages, num_kb)
    b_loads = [kb for kb in range(early_b)]                 # before pdl_wait: stage kb, expect_tx armed there
    expect = [kb for kb in range(early_b)]
    a_loads = []
    for kb in range(num_kb):                                # producer loop
        if kb >= early_b:
            expect.append(kb)
            b_loads.append(kb)
        a_loads.append(kb)
    assert b_loads == list(range(num_kb)) and a_loads == list(range(num_kb)) and expect == list(range(num_kb))
    assert all(kb % stages == kb for kb in range(early_b))  # early tiles land in the stage the loop will use
