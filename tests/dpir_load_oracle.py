"""ctypes binding of the CPU restatement of DoublePIR's init() and load_data (tests/cpp/dpir_load_oracle.cpp).  TEST
INFRASTRUCTURE ONLY: compiled on first import into a private temporary directory, removed again when the process exits, so
it writes nothing into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "cpp", "dpir_load_oracle.cpp")
_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _load():
    d = tempfile.mkdtemp(prefix="dpir_load_oracle_")
    atexit.register(shutil.rmtree, d, True)
    so = os.path.join(d, "libdpir_load_oracle.so")
    # OpenMP spreads derive_with_aes over its 64 KiB chunks
    subprocess.check_call([_CXX, "-O3", "-std=c++17", "-fPIC", "-fopenmp", "-Wall", "-Werror", "-shared", "-o", so, _SRC])
    lib = C.CDLL(so)
    lib.orc_load_last_error.restype = C.c_char_p
    u8p, u32p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    lib.orc_aes128_encrypt.argtypes = [C.c_char_p, C.c_char_p, u8p]
    lib.orc_dpir_derive_with_aes.argtypes = [C.c_char_p, u8p, C.c_size_t]
    lib.orc_dpir_db_info.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, u64p]
    lib.orc_dpir_load_data.argtypes = [u8p, C.c_size_t, C.c_int, C.c_uint64, C.c_uint64, C.c_size_t, C.c_size_t, C.c_uint64, u32p]
    return lib


LIB = _load()


def _ck(rc):
    if rc != 0:
        raise RuntimeError("oracle: " + LIB.orc_load_last_error().decode())


def _key(key):
    key = bytes(key)
    assert len(key) == 16
    return key


def aes128_encrypt(key, block):
    """FIPS-197 AES-128 of one 16-byte block."""
    block = bytes(block)
    assert len(block) == 16
    out = (C.c_uint8 * 16)()
    _ck(LIB.orc_aes128_encrypt(_key(key), block, out))
    return bytes(out)


def dpir_derive_with_aes(key, nbytes):
    """matrix/derivation.rs:11-22: nbytes of keystream (uint8 array)."""
    out = np.zeros(nbytes, dtype=np.uint8)
    _ck(LIB.orc_dpir_derive_with_aes(_key(key), out.ctypes.data_as(C.POINTER(C.c_uint8)), nbytes))
    return out


def dpir_derive_from_seed(rows, cols, key):
    """Matrix::derive_from_seed (matrix.rs:125-135): rows x cols u32, little-endian words of the keystream."""
    return dpir_derive_with_aes(key, rows * cols * 4).view("<u4").astype(np.uint32).reshape(rows, cols)


def dpir_db_info(num_entries, bits, p):
    """DbInfo::new (database.rs:58-90): dict(db_elems, packing, ne, x)."""
    out = np.zeros(4, dtype=np.uint64)
    _ck(LIB.orc_dpir_db_info(num_entries, bits, p, out.ctypes.data_as(C.POINTER(C.c_uint64))))
    return dict(zip(("db_elems", "packing", "ne", "x"), (int(v) for v in out)))


def dpir_load_data(data, bits_format, num_entries, bits, l, m, p):
    """Db::load_data (bits_format False: one entry a byte) / load_data_fast (True: eight a byte, LSB first), database.rs:168-247.
    Returns the l x m u32 matrix, or raises IndexError where the reference panics on an index past the matrix."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    out = np.zeros((l, m), dtype=np.uint32)
    rc = LIB.orc_dpir_load_data(data.ctypes.data_as(C.POINTER(C.c_uint8)), data.size, int(bits_format), num_entries, bits, l, m, p,
                                out.ctypes.data_as(C.POINTER(C.c_uint32)))
    if rc == 1:
        raise IndexError("load_data indexes past the %d x %d matrix" % (l, m))
    _ck(rc)
    return out
