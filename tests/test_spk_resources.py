"""CPU: resource usage of the speaker-measure kernels (csrc/spk.cu) in the built library (cuobjdump, no GPU needed).

Every kernel keeps its float64 accumulators in registers: a local-memory stack means ptxas spilled, and the score
tile's 16 accumulators would then round-trip through memory on every coordinate."""
import re
import subprocess

KERNELS = ("time_stats_kernel", "spk_norm_kernel", "spk_score_kernel", "spk_hist_kernel", "spk_step_kernel",
           "spk_result_kernel", "spk_group_mean_kernel")


def spk_resources():
    from adaptive_voice_conversion_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and any(k in fn for k in KERNELS) and "REG:" in line:
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


def test_spk_kernels_have_no_stack_and_no_spills():
    res = spk_resources()
    assert sorted(k for k in KERNELS if any(k in fn for fn in res)) == sorted(KERNELS), sorted(res)
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)


def test_step_kernel_fits_one_cta_of_1024_threads():
    for fn, r in spk_resources().items():
        if "spk_step_kernel" in fn:
            assert 1024 * r["REG"] <= 65536, (fn, r)
