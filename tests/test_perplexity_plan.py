"""The window plan of tools/perplexity.py: every target token is counted exactly once and no window is longer than the context."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def _tool():
    spec = importlib.util.spec_from_file_location("perplexity_tool", ROOT / "tools" / "perplexity.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("n,ctx,stride", [(2, 2, 1), (300, 128, 64), (300, 128, 127), (1000, 256, 1), (129, 128, 64), (128, 128, 64),
                                          (4097, 2048, 512), (50, 128, 64), (777, 100, 33)])
def test_window_plan_counts_each_target_once(n, ctx, stride):
    pp = _tool()
    plan = pp.window_plan(n, ctx, stride)
    tokens = np.arange(n) * 7 % 1000
    seen = np.zeros(n, dtype=int)
    for k, (start, length, first) in enumerate(plan):
        assert start == k * stride
        assert 2 <= length <= ctx and start + length <= n
        t = pp.window_targets(tokens, start, length, first)
        assert t.shape == (length,) and t[-1] == -1
        for i in np.nonzero(t >= 0)[0]:
            assert t[i] == tokens[start + i + 1]
            seen[start + i + 1] += 1
        if k:  # a later window counts only its last targets, at most `stride` of them
            assert 0 < int((t >= 0).sum()) <= stride
            assert np.all(t[:length - 1 - int((t >= 0).sum())] == -1)
    assert seen[0] == 0 and np.all(seen[1:] == 1)


@pytest.mark.parametrize("n,ctx,stride", [(1, 128, 64), (100, 128, 128), (100, 128, 0), (100, 1, 1)])
def test_window_plan_refuses(n, ctx, stride):
    with pytest.raises(ValueError):
        _tool().window_plan(n, ctx, stride)
