"""The fused x pass of the right-hand side (k_rfft_x_products) runs without local memory.

Its 224 KB shared-memory carve-out at n = 384 leaves the SM about 30 KB of L1, so every spill or stack-resident local of the
kernel turns into L2 traffic on its dependent chain.  This reads the compiled resource usage of every instance from the built
library (no GPU needed)."""
import pathlib, re, shutil, subprocess
import pytest

LIB = pathlib.Path(__file__).resolve().parents[1] / "dedalus_b200" / "libdedalus_b200.so"


def _resource_usage():
    if not LIB.exists():
        pytest.skip("libdedalus_b200.so has not been built")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "--dump-resource-usage", str(LIB)], capture_output=True, text=True, check=True).stdout
    usage, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            usage[fn] = (int(m.group(1)), int(m.group(2)))
            fn = None
    return usage


def test_x_products_have_no_stack_frame():
    usage = {fn: u for fn, u in _resource_usage().items() if "k_rfft_x_products" in fn}
    # n = 24, 48, 96, 192, 384, all at P = 8
    assert len(usage) == 5, sorted(usage)
    stacked = {fn: stack for fn, (_, stack) in usage.items() if stack != 0}
    assert not stacked, stacked
    for fn, (reg, _) in usage.items():
        assert reg <= 168, (fn, reg)
