"""tools/measure.py, the timing protocol of the A/B tools, on the host: the statistics, the order in which `alternate`
calls its arms, and that `tag_ms` always switches kernel timing off again."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("measure_under_test", os.path.join(ROOT, "tools", "measure.py"))
measure = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(measure)


def test_stats_odd_length_is_min_median_max():
    assert measure.stats([3.0, 1.0, 2.0]) == {"min": 1.0, "median": 2.0, "max": 3.0}


def test_stats_even_length_takes_the_upper_median_and_rounds():
    assert measure.stats([4.0, 1.0, 3.0, 2.0]) == {"min": 1.0, "median": 3.0, "max": 4.0}
    assert measure.stats([2.34567, 1.23456], nd=2) == {"min": 1.23, "median": 2.35, "max": 2.35}


def test_alternate_warms_up_every_arm_then_alternates(monkeypatch):
    calls, flushes = [], []

    def fake_timed(fn, flush=True):
        flushes.append(flush)
        out = fn()
        return out, float(len(calls))   # "ms": the call's position, so each sample names the call it came from

    def arm(name):
        def fn():
            calls.append(name)
            return f"{name}{len(calls)}"
        return fn

    monkeypatch.setattr(measure, "timed", fake_timed)
    ms, last = measure.alternate({"a": arm("a"), "b": arm("b")}, reps=3, warmup=2, flush=False)
    assert calls == ["a", "b"] * 2 + ["a", "b"] * 3
    assert flushes == [False] * 10
    assert ms == {"a": [5.0, 7.0, 9.0], "b": [6.0, 8.0, 10.0]}   # the warm-up calls are not in the samples
    assert last == {"a": "a9", "b": "b10"}


class FakeLib:
    def __init__(self):
        self.enabled, self.log = False, []

    def timing_enable(self, on):
        self.enabled = on
        self.log.append(("enable", on))

    def timing_collect(self):
        self.log.append(("collect", self.enabled))
        return {"tag": (1.5, 2)}


def test_tag_ms_collects_after_the_runs_while_timing_is_on(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(measure, "_lib", lib)
    runs = []
    assert measure.tag_ms(lambda: runs.append(lib.enabled), runs=3) == {"tag": (1.5, 2)}
    assert runs == [True] * 3
    assert lib.log == [("enable", True), ("collect", True), ("enable", False)]


def test_tag_ms_disables_timing_when_fn_raises(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(measure, "_lib", lib)

    def boom():
        raise RuntimeError("kernel failed")

    with pytest.raises(RuntimeError, match="kernel failed"):
        measure.tag_ms(boom, runs=2)
    assert lib.log == [("enable", True), ("enable", False)]
    assert not lib.enabled
