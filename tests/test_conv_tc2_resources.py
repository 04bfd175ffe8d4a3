"""CPU: resource usage of the persistent conv kernel in the built library (cuobjdump, no GPU needed).

Every instance of conv_block_tc2_kernel keeps its wgmma accumulators in registers: a local-memory stack means
ptxas spilled, and spilled accumulators serialise the asynchronous MMAs of the main loop."""
import re
import subprocess

TC2 = "conv_block_tc2_kernel"


def tc2_resources():
    from adaptive_voice_conversion_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and TC2 in fn and "REG:" in line:
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


def test_conv_tc2_kernel_has_no_stack():
    res = tc2_resources()
    # one instance per accumulator width (16..160), plus the chunked folded data-gradient widths
    assert len(res) >= 10, sorted(res)
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)


def test_conv_tc2_kernel_register_allocation_covers_setmaxnreg():
    # the block starts with REG registers per thread for 384 threads; setmaxnreg hands 56 to warpgroup 0 and 224 to
    # each consumer warpgroup, which must fit that allocation (otherwise setmaxnreg.inc waits forever)
    for fn, r in tc2_resources().items():
        assert 384 * r["REG"] >= 128 * 56 + 256 * 224, (fn, r)
