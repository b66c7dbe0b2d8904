"""NumPy statement of the sorted scan and the facet counts of OR-group and min-match queries
(sdbg_match_topk_by_column_batch_groups_min / sdbg_match_facet_counts_batch_groups_min): the docs
min_match_reference.match_docs gives per segment, sorted or counted per key exactly as sort_reference / facet_reference
do for the flat queries. Each segment's matching docs are handed to those references as the one list of a one-term
OR, with deletions, filter and exclusions already applied, so their order, NULL and key rules are reused as they are.

TEST INFRASTRUCTURE: imported by tests only."""
import facet_reference as fr
import min_match_reference as mr
import sort_reference as sr


def _as_one_term(seg_lists, groups, excl, deleted, masks, mins):
    """Per segment [the query's matching docs]: a one-term list set whose OR of term 0 is exactly the grouped query."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return [[mr.match_docs(l, groups, excl, d, m, mins)] for l, d, m in zip(seg_lists, deleted, masks)]


def sorted_hits(seg_lists, groups, columns, descending=False, nulls_first=False, k=None, excl=(), deleted=None, masks=None,
                mins=None):
    """sort_reference.sorted_hits of the query of OR groups `groups` (mins: per group its minimum, None: 1)."""
    return sr.sorted_hits(_as_one_term(seg_lists, groups, excl, deleted, masks, mins), "OR", [0], columns, descending,
                          nulls_first, k)


def facet_counts(seg_lists, groups, columns, key_min, key_span, excl=(), deleted=None, masks=None, mins=None):
    """facet_reference.facet_counts of the query of OR groups `groups`: (counts uint64[key_span], nulls)."""
    return fr.facet_counts(_as_one_term(seg_lists, groups, excl, deleted, masks, mins), "OR", [0], columns, key_min, key_span)


def facet_dict(seg_lists, groups, columns, excl=(), deleted=None, masks=None, mins=None):
    """facet_reference.facet_dict of the query of OR groups `groups`."""
    return fr.facet_dict(_as_one_term(seg_lists, groups, excl, deleted, masks, mins), "OR", [0], columns)
