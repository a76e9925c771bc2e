"""CPU: the index arithmetic the tensor-core kernels rely on, replayed in numpy -- shared-memory operand images
(K-major, 128-byte swizzle), the lane maps of the producers (forward GEMM, transposing TN GEMM) and of the wgmma accumulator.
Each test states the property the kernel comment claims (every element written exactly once; no shared-memory bank
conflicts inside a quarter-warp of a 128-bit access; coalesced 128-byte global segments) and checks it for all lanes."""
import numpy as np


def sw128_offset(row, chunk16):
    """Byte offset of the 16-byte chunk `chunk16` (4 fp32 of K) of image row `row`: rows are 128 B, the chunk index is
    XORed with row % 8 (SWIZZLE_128B) -- gemm_wgmma.cu / gemm_tn_wgmma.cu / pack_b_kernel."""
    return row * 128 + ((chunk16 ^ (row & 7)) << 4)


def bank_groups_16B(byte_offsets):
    return (np.asarray(byte_offsets) // 16) % 8          # 32 banks x 4 B = 8 groups of 16 B


def test_forward_producer_covers_the_tile_once_and_stores_without_conflicts():
    """gemm_wgmma_kernel A producers: f = ptid + i*128, row = f >> 3, c16 = f & 7 (i < 8, ptid < 128)."""
    seen = np.zeros((128, 8), dtype=int)
    for i in range(8):
        for warp in range(4):
            offs, glob = [], []
            for lane in range(32):
                f = warp * 32 + lane + i * 128
                row, c16 = f >> 3, f & 7
                seen[row, c16] += 1
                offs.append(sw128_offset(row, c16))
                glob.append((row, c16))
            offs = np.array(offs)
            for q in range(4):                            # a 128-bit store is issued per quarter-warp
                assert len(set(bank_groups_16B(offs[q * 8:(q + 1) * 8]))) == 8
            rows = {r for r, _ in glob}
            assert len(rows) == 4                         # one load instruction = 4 rows x 128 contiguous bytes of A
            for r in rows:
                assert sorted(c for rr, c in glob if rr == r) == list(range(8))
    assert np.all(seen == 1)


def test_transposing_producer_of_the_tn_gemm():
    """gemm_tn_wgmma_kernel: lane = l0 | c4 << 1 | gh << 3; image row (= matrix column) 32 w + 4 (l0 + 2 gh) + j;
    16-byte K chunk 4 h + c4; loads A[k0 + 16 h + 4 c4 + i][col .. col + 3]."""
    seen = np.zeros((128, 8), dtype=int)                  # image rows x 16-byte chunks of one 32-wide K step
    for w in range(4):
        for h in range(2):
            # loads: for fixed i, the 8 lanes that share c4 read 8 x 16 B = 128 contiguous bytes of one k row
            for i in range(4):
                by_k = {}
                for lane in range(32):
                    l0, c4, gh = lane & 1, (lane >> 1) & 3, lane >> 3
                    col = 32 * w + 4 * (l0 + 2 * gh)
                    k = 16 * h + 4 * c4 + i
                    by_k.setdefault(k, []).append(col)
                assert len(by_k) == 4
                for cols in by_k.values():
                    assert sorted(cols) == list(range(32 * w, 32 * w + 32, 4))
            # stores: for fixed j, every quarter-warp hits 8 distinct 16-byte bank groups
            for j in range(4):
                offs = []
                for lane in range(32):
                    l0, c4, gh = lane & 1, (lane >> 1) & 3, lane >> 3
                    row = 32 * w + 4 * (l0 + 2 * gh) + j
                    chunk = 4 * h + c4
                    seen[row, chunk] += 1
                    offs.append(sw128_offset(row, chunk))
                offs = np.array(offs)
                for q in range(4):
                    assert len(set(bank_groups_16B(offs[q * 8:(q + 1) * 8]))) == 8
    assert np.all(seen == 1)


def test_packed_weight_image_matches_the_operand_layout():
    """pack_b_kernel writes float index (nl >> 3) * 256 + (nl & 7) * 32 + ((c16 ^ (nl & 7)) << 2): the same byte address as
    sw128_offset(nl, c16), so a 1-D bulk copy of the image IS the shared-memory operand."""
    for nl in range(256):
        for c16 in range(8):
            assert 4 * ((nl >> 3) * 256 + (nl & 7) * 32 + ((c16 ^ (nl & 7)) << 2)) == sw128_offset(nl, c16)


def test_umma_k_step_advance_stays_inside_the_swizzle_atom():
    """The consumers advance the descriptor start address by 32 bytes per wgmma K = 8 tf32 (4 steps per 128-byte row):
    element (row, k) of k-step s must be found at base(s) + the swizzled position of (row, k - 8 s) computed with the
    address bits the hardware XORs (bits 4-6 with bits 7-9 of the absolute offset)."""
    def hw_address(base, row, kk):                        # 128B swizzle applied by the hardware on the absolute smem offset
        linear = base + row * 128 + kk * 4
        return linear ^ (((linear >> 7) & 7) << 4)
    for s in range(4):
        for row in range(16):
            for kk in range(8):
                want = sw128_offset(row, (8 * s + kk) // 4) + ((8 * s + kk) % 4) * 4
                assert hw_address(32 * s, row, kk) == want


def test_wgmma_accumulator_fragments_cover_the_tile_once():
    """epilogue_regs / the TN epilogue: thread t of a consumer warpgroup holds d[4 j + 2 i + e] of row 16 (t / 32) + (t % 32) / 4
    + 8 i and column 8 j + 2 (t % 4) + e -- every element of the 64 x BN accumulator exactly once, column pairs even-aligned."""
    for BN in (32, 64, 128):
        seen = np.zeros((64, BN), dtype=int)
        for t in range(128):
            for j in range(BN // 8):
                for i in range(2):
                    row, col = 16 * (t // 32) + (t % 32) // 4 + 8 * i, 8 * j + 2 * (t % 4)
                    assert col % 2 == 0
                    seen[row, col] += 1
                    seen[row, col + 1] += 1
        assert np.all(seen == 1)


def test_split_tf32_is_exact_and_three_products_recover_fp32_accuracy():
    """hi = x & 0xffffe000 is a TF32 value, lo = x - hi is exact in fp32; lo*hi + hi*lo + hi*hi drops only lo*lo (~2^-22)."""
    rng = np.random.default_rng(0)
    x = rng.standard_normal(4096).astype(np.float32)
    y = rng.standard_normal(4096).astype(np.float32)

    def split(v):
        hi = (v.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
        return hi, v - hi
    xh, xl = split(x); yh, yl = split(y)
    assert np.all((xh.view(np.uint32) & 0x1FFF) == 0)
    assert np.array_equal((xh.astype(np.float64) + xl.astype(np.float64)).astype(np.float32), x)       # exact decomposition
    lo_tf32 = (xl.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)                           # the tensor core truncates lo too
    ylo_tf32 = (yl.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    approx = lo_tf32.astype(np.float64) * yh + xh.astype(np.float64) * ylo_tf32 + xh.astype(np.float64) * yh
    exact = x.astype(np.float64) * y.astype(np.float64)
    rel = np.abs(approx - exact) / np.abs(exact).max()
    assert rel.max() < 2e-6                                                                             # vs ~5e-4 for one TF32 product
    one_pass = np.abs(xh.astype(np.float64) * yh - exact) / np.abs(exact).max()
    assert one_pass.max() > 1e-4


def packed_image_offset(BN, nl, c16):
    """pack_b_kernel: float index of the 16-byte chunk c16 of weight row nl (a column of B) inside one hi (or lo) image of BN rows."""
    return ((nl >> 3) * 256 + (nl & 7) * 32 + ((c16 ^ (nl & 7)) << 2)) * 4


def test_ring_stages_fit_the_shared_memory_of_an_sm90_block():
    """gemm_wgmma.cu: a stage holds the hi and lo images of A (128 rows) and of B (BN rows), 128 B per row; the ring takes what
    fits into 227 KB of opt-in shared memory less alignment slack and barriers, at most 4 stages -- and never fewer than the
    2 producer groups (test_producer_groups_never_exceed_ring_stages)."""
    ring_budget = 227 * 1024 - 1024 - 256                           # TC_RING_BUDGET
    stage = lambda bn: 2 * 128 * 128 + 2 * bn * 128                 # noqa: E731
    assert [min(4, ring_budget // stage(bn)) for bn in (32, 64, 128)] == [4, 4, 3]
    assert 3 * stage(128) + 1024 + 2 * 3 * 8 <= 227 * 1024


def test_producer_groups_never_exceed_ring_stages():
    """Why ngroups = min(TC_GROUPS, S): a group that published chunk q waits for the stage of chunk q + G.  The 'empty' barrier
    of that stage has completed the phases of all chunks <= the last one consumed; the consumer is at least at chunk q - S
    (the group could publish q).  The awaited phase is the one of chunk q + G - S; with G > S the barrier can still be two or
    more phases behind it, and a parity wait (1 bit) cannot distinguish 'two behind' from 'done'."""
    def phases_behind(G, S):
        worst = 0
        for q in range(S, 6 * S * G):
            awaited = (q + G - S) // S                      # use index (phase) of chunk q + G - S in its stage
            stage = (q + G) % S
            consumed_up_to = q - S                          # the consumer has at least finished chunk q - S
            done = max((c // S for c in range(stage, consumed_up_to + 1, S)), default=-1)   # last completed phase of that stage
            worst = max(worst, awaited - done)
        return worst
    for S in (2, 3, 4):
        for G in (1, 2, 3, 4):
            if G <= S:
                assert phases_behind(G, S) <= 1, (G, S)     # waiting for the very next phase: parity is unambiguous
            else:
                assert phases_behind(G, S) >= 2, (G, S)     # the bug of the first 3-group build (job C)
