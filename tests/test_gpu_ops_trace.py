"""The C calls of every ops wrapper, pinned: each case of tests/golden/make_ops_trace.py must make the same calls with the
same arguments in the same order, count the same launches and return the same tensors as when the fixture was recorded,
and a failing call must raise naming the symbol that was called.  The library is replaced by a recording stand-in, so
no kernel runs; the wrappers still need CUDA tensors."""
import json

import pytest

from tests.golden import make_ops_trace as trace

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    with open(trace.TRACE) as f:
        return json.load(f)


def test_cases_match_the_fixture(golden):
    assert sorted(trace.CASES) == sorted(golden)


@pytest.mark.parametrize("name", sorted(trace.CASES))
def test_call_trace(golden, name):
    got, _ = trace.run_case(trace.CASES[name])
    assert json.loads(json.dumps(got)) == golden[name]


@pytest.mark.parametrize("name", sorted(trace.CASES))
def test_failure_names_the_symbol_called(name):
    _, rec = trace.run_case(trace.CASES[name])
    launches = [c[0] for c in rec.calls if c[-1] == "stream"]
    for i, symbol in enumerate(launches):
        got, _ = trace.run_case(trace.CASES[name], fail_at=i)
        assert got["raises"] == ["RuntimeError", f"{symbol} failed: stand-in error ({trace.FAIL_CODE})"], (name, i)
        assert [c[0] for c in got["calls"] if c[-1] == "stream"] == launches[:i + 1]
