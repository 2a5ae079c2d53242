"""The eval-graph switch (no GPU): bts_b200.set_eval_graphs returns the previous setting and takes booleans only,
BTS_B200_EVAL_GRAPH sets the initial one (off when unset) and an invalid value fails the import.  A model's graph cache
is not carried into a deep copy or a pickle."""
import copy
import os
import pickle
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_set_eval_graphs_returns_the_previous_setting():
    import bts_b200
    start = bts_b200.get_eval_graphs()
    try:
        bts_b200.set_eval_graphs(False)
        assert bts_b200.set_eval_graphs(True) is False
        assert bts_b200.get_eval_graphs() is True
        assert bts_b200.set_eval_graphs(False) is True
        for bad in ("1", "on", None, 2):
            with pytest.raises(ValueError):
                bts_b200.set_eval_graphs(bad)
        assert bts_b200.get_eval_graphs() is False
    finally:
        bts_b200.set_eval_graphs(start)


def _import_with(value):
    env = dict(os.environ)
    env.pop("BTS_B200_EVAL_GRAPH", None)
    if value is not None:
        env["BTS_B200_EVAL_GRAPH"] = value
    code = "import sys; sys.path.insert(0, %r); import bts_b200; print(bts_b200.get_eval_graphs())" % ROOT
    return subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)


@pytest.mark.parametrize("value,on", [(None, "False"), ("0", "False"), ("1", "True")])
def test_environment_sets_the_initial_setting(value, on):
    r = _import_with(value)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip().splitlines()[-1] == on


@pytest.mark.parametrize("value", ["yes", "true", "2", ""])
def test_an_invalid_environment_value_fails_the_import(value):
    r = _import_with(value)
    assert r.returncode != 0
    assert "BTS_B200_EVAL_GRAPH" in r.stderr and repr(value) in r.stderr


def test_cache_is_not_copied_or_pickled():
    import torch
    from bts_b200 import graph
    m = torch.nn.Linear(2, 2)
    m._eval_graph_cache = graph._EvalGraphCache()
    m._eval_graph_cache.entries["key"] = object()            # stands for a captured graph, which cannot be copied
    for other in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert isinstance(other._eval_graph_cache, graph._EvalGraphCache)
        assert not other._eval_graph_cache.entries
        assert torch.equal(other.weight, m.weight)
