"""CPU: resource usage of the speaker-bank kernels in the built library (cuobjdump, no GPU needed).

The two pooling kernels keep their float4 sums and the identification kernel its float64 scores in registers: a
local-memory stack would mean ptxas spilled."""
import re
import subprocess

KERNELS = ("time_sum_varlen_kernel", "pooled_group_mean_kernel", "spk_identify_kernel")


def test_bank_kernels_have_no_stack_and_no_spills():
    from adaptive_voice_conversion_b200 import _lib as L
    L.load()
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and any(k in fn for k in KERNELS) and "REG:" in line:
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    assert sorted(k for k in KERNELS if any(k in fn for fn in res)) == sorted(KERNELS), sorted(res)
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)
