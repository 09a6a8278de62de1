"""The speculative-sampling acceptance rule (tests/spec_rule.py, the rule of include/tce_b200.h tce_spec_accept) on the CPU: it reduces to
the greedy rule at temp <= 0 and to the plain draw without drafts, and over fixed seeds its emitted path has the exact distribution of the
plain sampled loop."""
import numpy as np
import pytest
from scipy.stats import chisquare

from oracle import sampling
from spec_rule import accept_sampled, path_probs, row_chains

N_SEEDS = 20000


def _rows(V, d, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((d + 1, V)) * 2.0).astype(np.float32)


PEN_ON = dict(repeat_penalty=1.3, frequency_penalty=0.1, presence_penalty=0.05, repeat_last_n=8)
PEN_OFF = dict(repeat_penalty=1.0, frequency_penalty=0.0, presence_penalty=0.0, repeat_last_n=8)


@pytest.mark.parametrize("pen", [PEN_ON, PEN_OFF])
def test_greedy_at_temp_zero(pen):
    """temp <= 0: a draft is accepted exactly when it is the penalised arg-max, and the first rejected row emits its arg-max"""
    for case in range(40):
        V, d = 16 + case, 1 + case % 5
        rows = _rows(V, d, case)
        seq = [int(t) for t in np.random.default_rng(100 + case).integers(0, V, 6)]

        def greedy(j, drafts):
            win = ([0] * 8 + seq + drafts[:j])[-8:]
            return int(np.argmax(sampling.apply_penalties(rows[j], win, pen["repeat_penalty"], pen["frequency_penalty"], pen["presence_penalty"])))

        drafts = []
        for j in range(d):  # follow the arg-max for case % (d + 1) rows, then leave it
            g = greedy(j, drafts)
            drafts.append(g if j < case % (d + 1) else (g + 1) % V)
        k = 0
        while k < d and greedy(k, drafts) == drafts[k]:
            k += 1
        for seed in (0, 1, 12345):
            ids, acc, stop, q = accept_sampled(rows, drafts, seq, seed=seed, draw_index=len(seq), temp=0.0, **pen)
            assert ids == drafts[:k] + [greedy(k, drafts)] and acc == k and stop == 0, (case, seed)
            assert q.tolist() == [1.0] * k + [0.0] * (d + 1 - k)


@pytest.mark.parametrize("cfg", [dict(temp=0.7, top_k=40, top_p=0.9), dict(temp=1.5, top_k=5, top_p=1.0), dict(temp=0.2, top_k=0, top_p=0.95)])
def test_no_draft_is_the_plain_draw(cfg):
    for case in range(30):
        V = 16 + 2 * case
        rows = _rows(V, 0, 500 + case)
        seq = list(range(case % 7))
        ids_, probs = sampling.candidates(rows[0], ([0] * 8 + seq)[-8:], cfg["top_k"], cfg["top_p"], cfg["temp"], **{k: v for k, v in PEN_ON.items()
                                                                                                                     if k != "repeat_last_n"})
        for seed in range(20):
            ids, acc, stop, q = accept_sampled(rows, [], seq, seed=seed, draw_index=len(seq), **cfg, **PEN_ON)
            assert ids == [sampling.draw(ids_, probs, sampling.uniform01(seed, len(seq)))] and acc == 0 and q.tolist() == [0.0]


def _drafts(chains_fn, kind, V, d):
    """drafts whose row-j place among the candidates is `kind`: top, middle, tail candidate, or not a candidate"""
    drafts = []
    for j in range(d):
        ids, _ = chains_fn(drafts)[j]
        if kind == "top":
            drafts.append(int(ids[0]))
        elif kind == "middle":
            drafts.append(int(ids[ids.size // 2]))
        elif kind == "tail":
            drafts.append(int(ids[-1]))
        else:
            drafts.append(next(t for t in range(V) if t not in set(ids.tolist())))
    return drafts


def _chi2(counts, probs, n):
    """chi-square p-value of observed counts against exact probabilities, pooling outcomes expected fewer than 5 times"""
    keys = sorted(probs, key=lambda k: -probs[k])
    obs, exp, po, pe = [], [], 0, 0.0
    for k in keys:
        e = probs[k] * n
        if e >= 5:
            obs.append(counts.get(k, 0))
            exp.append(e)
        else:
            po += counts.get(k, 0)
            pe += e
    assert sum(counts.get(k, 0) for k in keys) == n, "an emitted path the rule cannot produce"
    if pe > 0:
        obs.append(po)
        exp.append(pe)
    if len(obs) < 2:
        return 1.0
    exp = np.array(exp) * (n / sum(exp))
    return float(chisquare(obs, exp).pvalue)


CASES = [
    # V, d, drafts kind, chain, penalties
    (16, 1, "top", dict(temp=0.7, top_k=40, top_p=1.0), PEN_OFF),
    (24, 2, "middle", dict(temp=1.5, top_k=12, top_p=1.0), PEN_ON),
    (32, 3, "tail", dict(temp=0.7, top_k=40, top_p=0.9), PEN_ON),
    (48, 2, "none", dict(temp=0.7, top_k=8, top_p=0.95), PEN_OFF),
    (64, 4, "top", dict(temp=1.0, top_k=0, top_p=1.0), PEN_ON),
    (40, 3, "middle", dict(temp=0.2, top_k=40, top_p=0.9), PEN_OFF),
]


@pytest.mark.parametrize("V,d,kind,cfg,pen", CASES)
def test_emitted_path_has_the_sampled_distribution(V, d, kind, cfg, pen):
    rows = _rows(V, d, V * 10 + d)
    rows[:, 0] += 1.0  # token 0 is in every zero-padded window: make the penalty matter
    seq = [3, 5, 3, 7]
    chains_fn = lambda drafts: row_chains(rows, drafts + [0] * (d - len(drafts)), seq, **cfg, **pen)
    drafts = _drafts(chains_fn, kind, V, d)
    chains = row_chains(rows, drafts, seq, **cfg, **pen)
    want = path_probs(chains, drafts)
    assert abs(sum(want.values()) - 1.0) < 1e-4
    counts, first = {}, {}
    for seed in range(N_SEEDS):
        ids, acc, stop, q = accept_sampled(rows, drafts, seq, seed=seed, draw_index=len(seq), chains=chains)
        key = (len(ids) - 1, ids[-1])
        assert ids[:-1] == drafts[:len(ids) - 1] and acc == len(ids) - 1
        counts[key] = counts.get(key, 0) + 1
        first[ids[0]] = first.get(ids[0], 0) + 1
    assert _chi2(counts, want, N_SEEDS) > 1e-3, (counts, want)
    p0 = {t: float(p) for t, p in zip(chains[0][0].tolist(), chains[0][1].tolist()) if p > 0}
    assert _chi2(first, p0, N_SEEDS) > 1e-3, (first, p0)
    if kind == "none":
        assert all(k == 0 for k, _ in counts)


def test_eos_and_budget_cut_the_step():
    V, d = 32, 4
    rows = _rows(V, d, 9)
    chains = [(np.array([7, 1, 2], dtype=np.int32), np.array([1.0, 0.0, 0.0], dtype=np.float32))] * (d + 1)  # q = 1 for draft 7: always accepted
    drafts = [7, 7, 7, 7]
    assert accept_sampled(rows, drafts, [], seed=1, draw_index=0, chains=chains)[:3] == ([7] * 5, 4, 0)
    assert accept_sampled(rows, drafts, [], seed=1, draw_index=0, chains=chains, budget=2)[:3] == ([7, 7], 2, 0)
    assert accept_sampled(rows, drafts, [], seed=1, draw_index=0, chains=chains, eos_id=7)[:3] == ([7], 1, 1)
