"""The device builds of the functor engines send their dense layers to library GEMMs (the wgmma kernels of gemm_tc.cu / gemm_ps.cu, cuBLAS SGEMM for weight
gradients); host emulation normally replaces them by functor GEMMs.  With NB200_EMU_LIBGEMM=1 the emulation shim takes the SAME dispatch
decisions as the device build and runs reference loops with the exact interface semantics of those libraries (strides, trans_b, accumulate,
bias; the cuBLAS argument order) -- so this run checks the ARGUMENTS the engines pass on the device path.  One representative test per engine,
in a subprocess (the switch is read once when the emulation library is loaded)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def test_engines_pass_correct_arguments_to_the_library_gemms():
    sel = ["tests/test_gemnet_emu.py::test_emu_matches_reference_golden_outputs",
           "tests/test_schnet_train_emu.py::test_schnet_energy_plus_force_loss_gradients_match_oracle_double_backward",
           "tests/test_gemnet_train_emu.py::test_small_batch_parameter_gradients_match_oracle_autograd"]
    p = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", *sel], cwd=os.path.dirname(HERE), capture_output=True, text=True,
                       timeout=1500, env=dict(os.environ, NB200_EMU_LIBGEMM="1"))
    assert p.returncode == 0 and "3 passed" in p.stdout, p.stdout[-2000:] + p.stderr[-1000:]
