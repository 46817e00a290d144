"""Point slices of the int8 digit-plane producer (i8_plane_slices in csrc/gram_i8_wgmma.cu), transcribed: the producer
splits a launch on its own, into the largest grid that runs in one wave at its shared-memory occupancy."""
import os
import re

TILE, PLANE_BYTES, UP = 128, 3 * 128 * 64, 64
H100_SXM_SMS = 132
SMEM_PER_SM, SMEM_RESERVED_PER_CTA = 228 * 1024, 1024      # sm_90: shared memory per SM, and the runtime's share per CTA


def plane_smem(d, direct=None):
    """Dynamic shared memory of the producer variant (launcher formula): tensor mode, or direct mode (n_terms, dpad4)."""
    if direct is None:
        nchunks = (3 * (-(-d // 16) * 16) + 16 + 63) // 64     # i8_nchunks
        xbytes, zbytes = nchunks * 8192, nchunks * 16384
    else:
        n_terms, dpad4 = direct
        xbytes, zbytes = n_terms * UP * dpad4 * 4, n_terms * TILE * dpad4 * 4
    return 1024 + 2 * PLANE_BYTES + zbytes + 4 * (xbytes + UP * 4) + 8 * 5


def plane_slices(m_pad, num_sms, n_units, smem):
    """The producer's point slices: the largest grid (tiles x slices) that fits one wave at the shared-memory occupancy."""
    per_sm = min(SMEM_PER_SM // (smem + SMEM_RESERVED_PER_CTA), 2048 // 256)
    return max(min(num_sms * per_sm // (m_pad // TILE), n_units), 1)


def test_producer_slices():
    units1, units3 = -(-1_000_000 // UP), -(-1_250_000 // UP)
    # configs[1]: d = 16, ~100 KB -> two CTAs per SM, 8 tiles x 33 slices = 264 CTAs (the Gram's split gave 88)
    assert plane_smem(16) < SMEM_PER_SM // 2 - SMEM_RESERVED_PER_CTA
    assert plane_slices(1024, H100_SXM_SMS, units1, plane_smem(16)) == 33
    # configs[3]: d = 32, one CTA per SM, 16 tiles x 8 slices = 128 CTAs in one wave
    assert plane_slices(2048, H100_SXM_SMS, units3, plane_smem(32)) == 8
    # more tiles than SM slots: one slice; fewer units than slices: one unit per slice
    assert plane_slices(128 * 300, H100_SXM_SMS, 10_000, plane_smem(16)) == 1
    assert plane_slices(128, H100_SXM_SMS, 5, plane_smem(16)) == 5


def test_producer_smem_formula_matches_source():
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc",
                            "gram_i8_wgmma.cu")).read()
    assert "*smem = 1024 + 2 * TILE_PLANES + *zbytes + XSTAGES * (*xbytes + UP * 4) + 8 * (XSTAGES + 1);" in src
    assert re.search(r"constexpr int XSTAGES = (\d+);", src).group(1) == "4"
    assert re.search(r"constexpr int NTHREADS = (\d+);", src).group(1) == "256"
