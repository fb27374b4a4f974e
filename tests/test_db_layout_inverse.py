"""CPU-only: the item maps of sdk_b200/csrc/item_place.cuh (where an item lives in database formats 0, 1 and 2, and how the
export kernels read it back) compiled with g++ and checked by tests/cpp/db_layout_inverse.cpp: fetch after place is the
identity for canonical residues, no two items share a byte, and unwritten cells read as zero."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_place_and_fetch_maps_are_mutually_inverse(tmp_path):
    exe = str(tmp_path / "db_layout_inverse")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "db_layout_inverse.cpp")])
    out = subprocess.check_output([exe], text=True)
    assert out.strip() == "layout maps ok", out
