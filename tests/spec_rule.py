"""numpy restatement of this project's speculative-sampling acceptance rule (include/tce_b200.h, tce_spec_accept) -- TEST INFRASTRUCTURE ONLY.

The reference has no speculative decoding, so this is not a restatement of reference code (that is what oracle/ holds): it is the rule the
header states, written out in float32 in the device's order, over the chain oracle.sampling restates.  `chains` lets a caller supply the
candidates and probabilities of each row (for instance the device sampler's own, read with tce_sample), so that the rule's arithmetic can
be compared bit for bit apart from the chain's exp().
"""
import numpy as np

from oracle.sampling import F, candidates, draw, uniform01

ACCEPT_STREAM = 0xD1B54A32D192ED03  # TCE_SPEC_ACCEPT_STREAM


def window(seq, drafts, j, repeat_last_n):
    """penalty window of row j: the last W entries of zeros ++ seq ++ drafts[:j], W = repeat_last_n (len(seq) when < 0)"""
    W = repeat_last_n if repeat_last_n >= 0 else len(seq)
    if W == 0:
        return []
    full = [0] * W + list(seq) + list(drafts[:j])
    return full[-W:]


def row_chains(rows, drafts, seq, *, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0,
               repeat_last_n=64):
    """(ids, probs) of every row under oracle.sampling.candidates"""
    return [candidates(rows[j], window(seq, drafts, j, repeat_last_n), top_k, top_p, temp, repeat_penalty, frequency_penalty, presence_penalty)
            for j in range(len(drafts) + 1)]


def row_rule(ids, probs, x, u):
    """-> (q, r) of one row: x the draft (None: no draft), u the draw uniform; r = -1 when the row counts as accepted with no replacement"""
    hit = np.nonzero(ids == x)[0] if x is not None else []
    q = F(probs[hit[0]]) if len(hit) else F(0.0)
    if q == F(0.0):
        return q, draw(ids, probs, u)
    ex = int(hit[0])
    S = F(0.0)
    for i in range(ids.size):
        if i != ex:
            S = F(S + probs[i])
    if S == F(0.0):
        return q, -1
    t = F(F(u) * S)
    run, r = F(0.0), -1
    for i in range(ids.size):
        if i == ex:
            continue
        run = F(run + probs[i])
        r = int(ids[i])
        if t < run:
            break
    return q, r


def accept_from_chains(chains, drafts, seed, draw_index, eos_id=-1, budget=None):
    """the rule over given per-row chains -> (ids, accepted, stop, q[rows])"""
    d = len(drafts)
    budget = d + 1 if budget is None else budget
    q, r = [], []
    for j, (ids, probs) in enumerate(chains):
        qj, rj = row_rule(ids, probs, int(drafts[j]) if j < d else None, uniform01(seed, draw_index + j))
        q.append(qj)
        r.append(rj)
    k = 0
    while k < d and (r[k] < 0 or F(uniform01(seed ^ ACCEPT_STREAM, draw_index + k)) < q[k]):
        k += 1
    out, stop = [], 0
    for i in range(k + 1):
        if len(out) >= budget:
            break
        t = int(drafts[i]) if i < k else r[k]
        out.append(t)
        if t == eos_id:
            stop = 1
            break
    return out, min(k, len(out)), stop, np.array(q, dtype=np.float32)


def accept_sampled(rows, drafts, seq, *, seed, draw_index, eos_id=-1, budget=None, chains=None, **cfg):
    """One speculative step: rows [d + 1][V] logits (row j after [last, drafts[:j]]), drafts d ids, seq the penalty sequence so far (h
    entries; the draw index of row j is draw_index + j, draw_index = h in the generate loop), cfg the tce_sampling fields.
    -> (emitted ids, accepted drafts among them, stop (eos_id emitted), q[d + 1])."""
    if chains is None:
        chains = row_chains(rows, drafts, seq, **cfg)
    return accept_from_chains(chains, drafts, seed, draw_index, eos_id, budget)


def path_probs(chains, drafts):
    """exact distribution of the emitted path (k, r_k): {(k, t): prod_{j<k} q_j * p_k(t)} with t != drafts[k] for k < d"""
    d = len(drafts)
    out, pre = {}, 1.0
    for k, (ids, probs) in enumerate(chains):
        for tok, p in zip(ids.tolist(), probs.tolist()):
            if (k < d and tok == int(drafts[k])) or pre * p <= 0:
                continue
            out[(k, tok)] = pre * p
        if k < d:
            hit = np.nonzero(ids == int(drafts[k]))[0]
            pre *= float(probs[hit[0]]) if len(hit) else 0.0
    return out
