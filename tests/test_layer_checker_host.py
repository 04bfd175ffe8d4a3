"""The layer tap's error bookkeeping (test_gpu_step_layers.Checker), which needs no GPU: a NaN error stays the worst of
its kind, so one NaN sample or group among finite ones fails its bound."""
import math

from test_gpu_step_layers import Checker


def test_nan_stays_the_worst():
    chk = Checker(None, {}, {}, False)
    for unit, e in (("a", 1e-7), ("b", float("nan")), ("c", 3e-7), ("d", 0.0)):
        chk.err("misc", unit, e)
    assert math.isnan(chk.worst["misc"]) and chk.where["misc"] == "b"
    chk.err("fwd", "first", float("nan"))
    chk.err("fwd", "second", 1.0)
    assert math.isnan(chk.worst["fwd"]) and chk.where["fwd"] == "first"


def test_first_error_names_its_unit():
    chk = Checker(None, {}, {}, False)
    chk.err("misc", "exact", 0.0)
    chk.err("misc", "also exact", 0.0)
    chk.err("dw", "x", 2e-7)
    chk.err("dw", "y", 1e-7)
    chk.err("dw", "z", 5e-7)
    assert (chk.worst["misc"], chk.where["misc"]) == (0.0, "exact")
    assert (chk.worst["dw"], chk.where["dw"]) == (5e-7, "z")
