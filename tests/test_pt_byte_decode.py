"""CPU-only: the plaintext decode rule of sdk_b200/csrc/item_place.cuh (pt_byte_decode, the inverse of convert_pt_to_poly's
recenter_mod that the item reader k_read_items applies to every coefficient) compiled with g++ and checked by
tests/cpp/pt_byte_decode.cpp: all 256 bytes round-trip, every other residue pair is rejected, and words that are not
canonical residues decode as their residue."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pt_byte_decode_inverts_recenter_mod_exactly(tmp_path):
    exe = str(tmp_path / "pt_byte_decode")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "pt_byte_decode.cpp")])
    out = subprocess.check_output([exe], text=True)
    assert out.strip() == "decode rule ok", out
