"""tests/cpp/dpir_tc_emul.cpp: the operand images, unpacking and epilogue of DoublePIR's tensor-core pass (dpir_tc.cu), run
thread by thread and lane by lane on the CPU through the index maps of dpir_tc_layout.cuh, with the wgmma replaced by the
definitions of the no-swizzle K-major layout and the accumulator fragment, against the 64-bit matrix_mul_vec_packed."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dpir_tc_pass_emulation(tmp_path):
    exe = str(tmp_path / "dpir_tc_emul")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-O2", "-std=c++17", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "dpir_tc_emul.cpp")])
    out = subprocess.check_output([exe], text=True)
    assert out.strip() == "dpir tc emulation ok", out
