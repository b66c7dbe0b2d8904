"""NumPy statement of minimum match counts over OR groups of phrases and terms (sdbg_phrase_groups_*_batch_min), built on
phrase_groups_reference.py without changing it, the way min_match_reference.py builds on groups_reference.py.

Everything is as phrase_groups_reference states it, with one addition: positive group g holds doc d when at least
mins[g] of its alternatives have phrase frequency > 0 in d (mins None: 1 for every group, which is exactly the
phrase_groups_reference statement). Every alternative counts on its own, so duplicate alternatives each count. A negated
group keeps minimum 1. The score is unchanged: the sum over every positive alternative with frequency > 0, so a doc that
holds more than mins[g] alternatives of a group is scored on all of them (IResearch's min-match disjunction scores so).
Only `match` / `matches` are new; scores and the passes are phrase_groups_reference's.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import phrase_groups_reference as pgr
import phrase_reference as pr

flat = pgr.flat
cost_order = pgr.cost_order
scores = pgr.scores
topk = pgr.topk
count = pgr.count
sorted_hits = pgr.sorted_hits
facet_counts = pgr.facet_counts
aggregate = pgr.aggregate
scan = pgr.scan


def match(docs, groups, excl=(), deleted=None, mask=None, mins=None):
    """(doc ids, per doc the phrase frequencies of every alternative, flattened) of one segment's matches, by doc; mins:
    one minimum per group (None: all 1; negated groups must have 1)."""
    mins = [1] * len(groups) if mins is None else list(mins)
    assert len(mins) == len(groups)
    for (alts, neg), m in zip(groups, mins):
        assert 1 <= m <= len(alts) and (m == 1 or not neg)
    dels = set() if deleted is None else {int(d) for d in deleted}
    ex = {int(t) for t in excl}
    ds, fs = [], []
    for i, seq in enumerate(docs):
        d = i + 1
        if d in dels or (mask is not None and not mask[i]) or ex.intersection(seq):
            continue
        f, ok = [], True
        for (alts, neg), m in zip(groups, mins):
            g = [pr.phrase_freq(seq, terms, rel) for terms, rel in alts]
            f += g
            held = sum(1 for x in g if x > 0)
            ok = ok and (held == 0 if neg else held >= m)
        if ok:
            ds.append(d)
            fs.append(f)
    return np.array(ds, np.uint32), fs


def matches(seg_docs, groups, excl=(), deleted=None, masks=None, mins=None):
    n = len(seg_docs)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return [match(d, groups, excl, x, m, mins) for d, x, m in zip(seg_docs, deleted, masks)]
