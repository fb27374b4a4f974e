"""CPU-only: the host parser of /update-row bodies (sdk_b200/csrc/update_body.hpp, run through tests/cpp/update_body_check.cpp)
against the entry-by-entry restatement of update_many_items (tests/update_rows_oracle.py): offsets, lengths, where the valid
prefix ends, the first error, largest_update, and which occurrence of a repeated db_idx survives."""
import os
import subprocess

import numpy as np
import pytest

import update_rows_oracle as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_CHUNK, NUM_ITEMS = 4 + 4 * 2048, 256          # parameter set T: 4 slices x 2048 bytes per chunk, 64 x 4 items


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ubc") / "update_body_check")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-O1", "-std=c++17", "-Wall", "-Werror",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "update_body_check.cpp")])
    return exe


def _run(checker, tmp_path, body):
    path = tmp_path / "body.bin"
    path.write_bytes(bytes(body))
    out = subprocess.check_output([checker, str(path), str(MAX_CHUNK), str(NUM_ITEMS)], text=True).split("\n")
    err = int(out[0].split()[1])
    largest = int(out[1].split()[1])
    entries = [tuple(int(x) for x in ln.split()[1:]) for ln in out if ln.startswith("entry ")]
    kept = [int(ln.split()[1]) for ln in out if ln.startswith("kept ")]
    return err, largest, entries, kept


def _expected_kept(entries):
    last = {}
    for pos, _, idx in entries:
        last[idx] = pos
    return sorted(last.values())


def _bodies():
    rng = np.random.default_rng(5)
    full = rng.integers(0, 256, MAX_CHUNK - 4, dtype=np.uint8)
    good = U.entry(7, full) + U.entry(0, full[:100]) + U.entry(NUM_ITEMS - 1, b"") + U.entry(7, full[:3]) + U.entry(9, full[:1])
    yield "empty", b""
    yield "good", good
    yield "one idx three times", U.entry(5, full[:10]) + U.entry(6, full[:20]) + U.entry(5, full[:30]) + U.entry(5, full[:40])
    yield "header truncated", good + b"\x00\x00"
    yield "header truncated at 3", good + b"\x00\x00\x10"
    yield "chunk truncated", good + U.entry(3, full[:50])[:-1]
    yield "chunk_len 0", good + (0).to_bytes(4, "big") + U.entry(1, b"")
    yield "chunk_len 3", good + (3).to_bytes(4, "big") + b"\x00\x00\x00" + U.entry(1, b"")
    yield "over-long", good + U.entry(2, np.zeros(MAX_CHUNK - 3, dtype=np.uint8)) + U.entry(1, b"")
    yield "longest allowed", U.entry(2, np.zeros(MAX_CHUNK - 4, dtype=np.uint8))
    yield "bad db_idx", good + U.entry(NUM_ITEMS, b"\x01") + U.entry(1, b"")
    yield "db_idx 2^32-1", U.entry(0xFFFFFFFF, b"")
    yield "chunk_len 2^32-1", (0xFFFFFFFF).to_bytes(4, "big") + b"\x00" * 16
    for k in range(20):                                           # random walks with a random corruption
        parts = [U.entry(int(rng.integers(0, NUM_ITEMS)), full[:int(rng.integers(0, 300))]) for _ in range(int(rng.integers(1, 12)))]
        b = bytearray(b"".join(parts))
        if k % 2:
            b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
        yield "random %d" % k, bytes(b)


def test_cpp_mirror_program_compiles_and_links(tmp_path):
    """tests/cpp/update_many_mirror.cpp (run on the GPU by test_gpu_update_many.py) builds against include/b200pir.hpp here."""
    from sdk_b200 import build
    build.build()
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o",
                           str(tmp_path / "update_many_mirror"), os.path.join(ROOT, "tests", "cpp", "update_many_mirror.cpp"),
                           "-L" + os.path.join(ROOT, "sdk_b200"), "-lb200pir", "-Wl,-rpath," + os.path.join(ROOT, "sdk_b200")])


@pytest.mark.parametrize("name,body", list(_bodies()), ids=[n for n, _ in _bodies()])
def test_parser_matches_update_many_items_walk(checker, tmp_path, name, body):
    err, largest, entries, kept = _run(checker, tmp_path, body)
    ref_entries, ref_err, ref_largest = U.walk(body, MAX_CHUNK, NUM_ITEMS)
    assert entries == ref_entries, name
    assert (err != 0) == (ref_err is not None), (name, err, ref_err)
    if ref_err is not None:
        assert err == -2, name                                    # B200PIR_E_SHAPE
    assert largest == ref_largest, name
    assert kept == _expected_kept(ref_entries), name
