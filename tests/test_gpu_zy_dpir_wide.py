"""DoublePIR's short-and-wide database shape (SURVEY 8d config #4, second case): the reference's own end-to-end test uses 2^24
one-bit entries, which approx_database_dims lays out as l = 29 rows x m = 65536 columns (doublepir.rs:471-483,
database.rs:376-418): 21846 packed words per row, more than fits beside `b` in shared memory, served by the wide-row kernel.
Sorted late: added after the last GPU session of the round."""
import numpy as np
import pytest

import oracle_lib as O
from test_gpu_parity import _gpu

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("rows,cols", [(29, 21846), (32, 17067), (3, 40001), (1, 17068)])
def test_dpir_matvec_wide_rows_match_oracle(rows, cols):
    _gpu()
    import sdk_b200.doublepir as D
    rng = np.random.default_rng(rows * 7 + cols)
    a = rng.integers(0, 2**30, rows * cols, dtype=np.uint32)
    a[:cols] = 0x3FFFFFFF                                       # first row: every 10-bit field at its maximum
    b = rng.integers(0, 2**32, 3 * cols, dtype=np.uint32)
    b[:7] = 0xFFFFFFFF
    m = D.PackedMatrix(a, rows, cols)
    try:
        assert np.array_equal(D.matrix_mul_vec_packed(m, b), O.dpir_matvec_packed(a, b, rows, cols))
    finally:
        m.close()


def test_dpir_limb_gemm_with_wrapping_accumulators():
    """The limb GEMM keeps four s32 register accumulators; with K beyond 2^15 and extreme operands they wrap.  Only the sum modulo
    2^32 is wanted, and a wrapped accumulator is still exact modulo 2^32 (DESIGN 4.5): K = 70016 with rows of all-255, all -2^15,
    all 2^15 - 1 against columns of 0xffffffff."""
    _gpu()
    import sdk_b200.doublepir as D
    rows, kdim, cols = 64, 70016, 64
    rng = np.random.default_rng(5)
    a = (rng.integers(0, 1024, (rows, kdim)).astype(np.int64) - 512).astype(np.uint32)
    a[0, :] = 255
    a[1, :] = np.uint32(2**32 - 32768)
    a[2, :] = 32767
    b = rng.integers(0, 2**32, (kdim, cols), dtype=np.uint64).astype(np.uint32)
    b[:, 0] = 0xFFFFFFFF
    b[:, 1] = 0x00FF00FF
    assert np.array_equal(D.matmul(a, b), O.dpir_mul(a, b, rows, kdim, cols))
