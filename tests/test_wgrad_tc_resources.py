"""CPU: resource usage of the wgmma weight-gradient kernel in the built library (cuobjdump, no GPU needed).

Every instance of conv_wgrad_wgmma_kernel (one per tap count and output mode) keeps its N / 2 <= 128 accumulators in
registers: a local-memory stack means ptxas spilled, and spilled accumulators serialise the asynchronous MMAs.  The
kernel runs 384 threads per block with no register split between the roles, so every instance must fit the 168
registers per thread of its __launch_bounds__ cap."""
import re
import subprocess

WG = "conv_wgrad_wgmma_kernel"


def wgrad_resources():
    from adaptive_voice_conversion_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and WG in fn and "REG:" in line:
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


def test_wgrad_wgmma_kernel_has_no_stack():
    res = wgrad_resources()
    assert len(res) == 16, sorted(res)   # K = 1..8, scratch and accumulate variants
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)
        assert r["REG"] <= 168, (fn, r)


def test_mma_sync_weight_gradient_kernel_is_gone():
    from adaptive_voice_conversion_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    assert "conv_wgrad_split_kernel" not in out
