"""The oracle's restatement of DoublePIR's init() and load_data (tests/cpp/dpir_load_oracle.cpp), which the GPU load is compared with.

AES-128 is third-party arithmetic here (the reference uses the `aes` and `ctr` crates), so it is pinned to FIPS-197 and
SP 800-38A, to the reference's own derive_with_aes_is_correct bytes (matrix/derivation.rs:69-85) and, where the
`cryptography` package is importable, to its AES-CTR.  DbInfo::new and load_data / load_data_fast are pinned to the numpy
restatement in test_oracle_doublepir_e2e.py."""
import hashlib

import numpy as np
import pytest

import dpir_load_oracle as L
import test_oracle_doublepir_e2e as E

SEED_A1 = bytes.fromhex("9c22778545ac229741908e652d333a0f")      # util/consts.rs:23-33
SEED_A2 = bytes.fromhex("5fffc482c72a854a10359e9fa2f5e07f")


def test_aes128_fips197_appendix_c1():
    key = bytes(range(16))
    assert L.aes128_encrypt(key, bytes.fromhex("00112233445566778899aabbccddeeff")).hex() == "69c4e0d86a7b0430d8cdb78070b4c55a"


def test_aes128_ctr_sp800_38a_f51():
    # F.5.1 CTR-AES128.Encrypt: keystream block k = AES(counter block k); the counter's low 64 bits never carry here, so
    # Ctr64BE (the reference's counter) gives the same blocks
    key = bytes.fromhex("2b7e151628aed2a6abf7158809cf4f3c")
    ctr = int("f0f1f2f3f4f5f6f7f8f9fafbfcfdfeff", 16)
    pts = ["6bc1bee22e409f96e93d7e117393172a", "ae2d8a571e03ac9c9eb76fac45af8e51", "30c81c46a35ce411e5fbc1191a0a52ef",
           "f69f2445df4f9b17ad2b417be66c3710"]
    cts = ["874d6191b620e3261bef6864990db6ce", "9806f66b7970fdff8617187bb9fffdff", "5ae4df3edbd5d35e5b4f09020db03eab",
           "1e031dda2fbe03d1792170a0f3009cee"]
    for k, (pt, ct) in enumerate(zip(pts, cts)):
        block = ((ctr & ~((1 << 64) - 1)) | ((ctr + k) & ((1 << 64) - 1))).to_bytes(16, "big")
        ks = L.aes128_encrypt(key, block)
        assert bytes(a ^ b for a, b in zip(ks, bytes.fromhex(pt))).hex() == ct, k


def test_seeds_are_sha256_prefixes():
    assert SEED_A1 == hashlib.sha256(b"blyss1").digest()[:16]
    assert SEED_A2 == hashlib.sha256(b"blyss2").digest()[:16]


def test_derive_with_aes_reference_bytes():
    d = L.dpir_derive_with_aes(SEED_A1, 265 * 65536)                  # derivation.rs:69-85 derive_with_aes_is_correct
    assert (d[0], d[16], d[258 * 65536]) == (247, 196, 63)
    d = L.dpir_derive_with_aes(SEED_A2, 265 * 65536)
    assert (d[0], d[258 * 65536]) == (132, 254)


@pytest.mark.parametrize("key", [SEED_A1, SEED_A2])
def test_derive_with_aes_equals_cryptography_ctr(key):
    ciphers = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    nbytes = 3 * 65536 + 100                                          # a partial last chunk ending in a partial block
    got = L.dpir_derive_with_aes(key, nbytes).tobytes()
    want = b""
    for i in range((nbytes + 65535) // 65536):
        enc = ciphers.Cipher(ciphers.algorithms.AES(key), ciphers.modes.CTR(i.to_bytes(8, "big") + bytes(8))).encryptor()
        want += enc.update(bytes(min(65536, nbytes - 65536 * i))) + enc.finalize()
    assert got == want


def test_derive_from_seed_reads_little_endian_words():
    d = L.dpir_derive_with_aes(SEED_A1, 7 * 3 * 4)
    m = L.dpir_derive_from_seed(7, 3, SEED_A1)
    assert m.shape == (7, 3) and m[0, 0] == int.from_bytes(d[:4].tobytes(), "little")
    assert np.array_equal(m.reshape(-1), d.view("<u4"))


@pytest.mark.parametrize("num_entries,bits,p", [(1 << 24, 1, 512), (1 << 20, 10, 512), (1000, 3, 512), (300, 8, 16), (5, 63, 2),
                                                 (77, 9, 1024), (77, 10, 1023), (12, 4, 17), (1 << 33, 1, 512)])
def test_db_info_equals_numpy(num_entries, bits, p):
    db_elems, ne, packing = E.num_db_entries(num_entries, bits, p)
    assert L.dpir_db_info(num_entries, bits, p) == dict(db_elems=db_elems, packing=packing, ne=ne, x=ne)


def _entries(data, bits_format):
    return np.unpackbits(data, bitorder="little") if bits_format else data


# (num_entries, bits, p, l, m, bytes, data high): packing with a partial last group; ne > 1 (p = 16, 8-bit entries);
# oversized byte entries (values up to 255 in 3-bit fields spill into the next field); a database with untouched words
LAYOUTS = [(1000, 1, 512, 2, 64, 1000, 2), (300, 8, 16, 10, 64, 300, 256), (999, 3, 512, 6, 64, 999, 256),
           (130, 10, 512, 10, 32, 130, 256), (9, 1, 512, 3, 7, 9, 2)]


@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m,nbytes,high", LAYOUTS)
def test_load_data_equals_numpy(num_entries, bits, p, l, m, nbytes, high, bits_format):
    rng = np.random.default_rng(num_entries * 7 + bits)
    nbytes = (nbytes + 7) // 8 if bits_format else nbytes
    data = rng.integers(0, 256 if bits_format else high, nbytes, dtype=np.uint8)
    entries = _entries(data, bits_format)
    prm = dict(l=l, m=m, p=p, logq=32)
    _, want = E.db_with_data(len(entries), bits, prm, entries)
    got = L.dpir_load_data(data, bits_format, num_entries, bits, l, m, p)
    assert np.array_equal(got, want)
    assert got[-1, -1] == np.uint32((-(p // 2)) % (1 << 32))            # untouched words are 0 - p/2 too


@pytest.mark.parametrize("bits_format", [False, True])
def test_load_data_overrun_raises(bits_format):
    # packing 9: 2 x 4 elements hold 72 entries, one more overruns; ne = 2 (p = 16, 8 bits): 2 rows of 4 hold 4 entries
    for count, bits, p, l, m in [(73, 1, 512, 2, 4), (5, 8, 16, 2, 4)]:
        nb = count
        if bits_format:
            nb = (count + 7) // 8
            count = 8 * nb
        data = np.ones(nb, dtype=np.uint8)
        with pytest.raises(IndexError):
            L.dpir_load_data(data, bits_format, 1, bits, l, m, p)
    # exactly full does not raise
    L.dpir_load_data(np.ones(72 // (8 if bits_format else 1), dtype=np.uint8), bits_format, 1, 1, 2, 4, 512)
