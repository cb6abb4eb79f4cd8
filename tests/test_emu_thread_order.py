"""The kernel emulation schedules the threads of a block cooperatively, lowest thread first.  Code that is correct only because of
that order -- a missing __syncthreads / __syncwarp between a producer and a consumer -- would still pass; DB_EMU_ORDER=reverse runs
the threads in descending order instead, so such code fails in one of the two orders.  This re-runs the tests of the kernels that have
not been on hardware (dense shell systems, pair combinations with radial symbols, matsolver plugins) and of the banded kernels in
reverse order; the whole CPU suite passes that way too (run it with the variable set).  The same subprocess style re-runs the kernel
variants behind environment switches and the cp.async kernels with the other landing model of the emulated copies (DB_EMU_CP)."""
import os, subprocess, sys, pathlib
ROOT = pathlib.Path(__file__).resolve().parents[1]


def test_kernels_pass_with_reversed_thread_order():
    env = dict(os.environ, DB_EMU_ORDER="reverse")
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider",
           str(ROOT / "tests" / "test_emu_shell.py"), str(ROOT / "tests" / "test_emu_sphere.py"), str(ROOT / "tests" / "test_emu_plugins.py"),
           str(ROOT / "tests" / "test_emu_banded.py"), str(ROOT / "tests" / "test_emu_pencil_batches.py"),
           "-k", "a_sbdf2 or banded or sw16 or matsolver or transforms or pencil_batches"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env, cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout


def test_alternative_kernel_variants():
    """The dense solve with its columns in global memory (taken for n > 800, selected here at small n with DB_DENSE_SOLVE_SMEM=0)
    stays correct."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider",
           str(ROOT / "tests" / "test_emu_shell.py"), str(ROOT / "tests" / "test_emu_sphere.py"), "-k", "dense or a_sbdf2"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, DB_DENSE_SOLVE_SMEM="0"), cwd=str(ROOT))
    assert out.returncode == 0 and " passed" in out.stdout, out.stdout[-3000:] + out.stderr[-2000:]


def test_cp_async_kernels_pass_with_copies_landing_at_issue():
    """The emulation lands a cp.async copy when a wait retires its group (DB_EMU_CP=late, the default of every other test), which
    catches reads before the copy has landed.  DB_EMU_CP=early lands it at issue instead, which catches the opposite mistake: a buffer
    refilled while other code still reads the previous contents.  This re-runs the kernels that use cp.async that way: the
    pointwise programs (k_pointwise_v3, k_pointwise_pairs inside the solvers), the four register-resident FFT kernels, the
    pipelined pencil solve's gather (DB_SOLVE_PIPE=1), and the banded kernels."""
    tests = ROOT / "tests"
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider",
           str(tests / "test_emu_banded.py"), str(tests / "test_emu_pencil.py"), str(tests / "test_emu_transforms.py"),
           str(tests / "test_emu_sphere.py"), str(tests / "test_emu_solver.py"), str(tests / "test_emu_pencil_batches.py"),
           "-k", "banded or sw16 or pencil_kernels or pointwise or register or benchmark_line or blocked_row or rb3d_steps or pipelined"
                 " or pencil_batches"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, DB_EMU_CP="early"), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout


def test_pencil_batches_pass_with_bulk_copies_landing_at_issue():
    """The emulation lands a bulk copy when a thread waits on its mbarrier (DB_EMU_BULK=late, the default), which catches a ring stage
    read before its wait.  DB_EMU_BULK=early lands it at issue, which catches a stage refilled while it is still being read."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", str(ROOT / "tests" / "test_emu_pencil_batches.py"),
           str(ROOT / "tests" / "test_emu_pencil.py"), "-k", "pencil_batches or merged"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, DB_EMU_BULK="early"), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout
