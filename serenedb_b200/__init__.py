"""serenedb_b200 -- H100-native (sm_90a) implementation of SereneDB's query-time hot path:
IResearch BM25 posting scan + top-k, and the `iresearch_scan` columnar filter -> aggregate.

The package is a thin host layer over libsdbg.so (hand-written CUDA behind the C ABI in
include/sdbg.h). Importing it loads the native library; if the library cannot be built or loaded the
import raises -- there is no Python or CPU fallback for any operation.
"""
from . import _native
from .engine import (ExecuteDistCountGroupsBatch, ExecuteDistFacetCountsGroupsBatch, ExecuteDistMatchAggregatesGroupsBatch,
                     ExecuteDistTopKByColumnGroupsBatch, MatchAggregatesDevice, TopKByColumnDevice, match_aggregate_device_bytes,
                     merge_aggregates_gathered, merge_topk_by_column_gathered, topk_by_column_device_bytes)
from .engine import ExecuteDistTopKGroupsBatch, TopKGroupsDevice, merge_topk_groups_gathered, topk_groups_device_bytes
from .engine import ExecutePhraseCount, ExecutePhraseCountBatch, ExecutePhraseTopK, ExecutePhraseTopKBatch
from .engine import (ExecutePhraseTopKByColumn, ExecutePhraseTopKByColumnBatch, ExecutePhraseFacetCounts,
                     ExecutePhraseFacetCountsBatch, ExecutePhraseMatchAggregates, ExecutePhraseMatchAggregatesBatch,
                     ExecutePhraseMatchScan, ExecutePhraseMatchScanBatch)
from .engine import (ExecutePhraseAndCount, ExecutePhraseAndCountBatch, ExecutePhraseAndTopK, ExecutePhraseAndTopKBatch, ExecutePhraseAndTopKByColumn, ExecutePhraseAndTopKByColumnBatch,
                     ExecutePhraseAndFacetCounts, ExecutePhraseAndFacetCountsBatch, ExecutePhraseAndMatchAggregates, ExecutePhraseAndMatchAggregatesBatch, ExecutePhraseAndMatchScan, ExecutePhraseAndMatchScanBatch)
from .engine import (ExecutePhraseGroupsCount, ExecutePhraseGroupsCountBatch, ExecutePhraseGroupsTopK, ExecutePhraseGroupsTopKBatch,
                     ExecutePhraseGroupsTopKByColumn, ExecutePhraseGroupsTopKByColumnBatch, ExecutePhraseGroupsFacetCounts,
                     ExecutePhraseGroupsFacetCountsBatch, ExecutePhraseGroupsMatchAggregates, ExecutePhraseGroupsMatchAggregatesBatch,
                     ExecutePhraseGroupsMatchScan, ExecutePhraseGroupsMatchScanBatch)
from .engine import (AND, OR, BM25, TFIDF, FLT_MIN, Context, ExecuteCount, ExecuteCountBatch, ExecuteCountGroups,
                     ExecuteCountGroupsBatch, ExecuteFacetCounts, ExecuteFacetCountsBatch, ExecuteFacetCountsGroups,
                     ExecuteFacetCountsGroupsBatch, ExecuteMatchAggregates, ExecuteMatchAggregatesBatch,
                     ExecuteMatchAggregatesGroups, ExecuteMatchAggregatesGroupsBatch, ExecuteMatchScanBatch, ExecuteMatchScanGroupsBatch, ExecuteTopK, ExecuteTopKBatch, ExecuteTopKByColumn, ExecuteTopKByColumnBatch,
                     ExecuteTopKByColumnGroups, ExecuteTopKByColumnGroupsBatch, ExecuteTopKGroups, ExecuteTopKGroupsBatch, IndexReader, IResearchScan, PostingsWriter, PreparedBatch, Segment, merge_gathered, pred,
                     resolve_pred, stage_parse_host, sum_i128, StreamScoredDocs, pack_for)

_native.lib()  # fail loudly at import time when the CUDA extension is missing

__all__ = ["AND", "OR", "BM25", "TFIDF", "FLT_MIN", "Context", "ExecuteCount", "ExecuteCountBatch", "ExecuteCountGroups",
           "ExecuteCountGroupsBatch", "ExecuteFacetCounts", "ExecuteFacetCountsBatch", "ExecuteFacetCountsGroups",
           "ExecuteFacetCountsGroupsBatch", "ExecuteMatchAggregates", "ExecuteMatchAggregatesBatch",
           "ExecuteMatchAggregatesGroups", "ExecuteMatchAggregatesGroupsBatch", "ExecuteMatchScanBatch", "ExecuteMatchScanGroupsBatch", "ExecuteTopK", "ExecuteTopKBatch", "ExecuteTopKByColumn", "ExecuteTopKByColumnBatch",
           "ExecuteTopKByColumnGroups", "ExecuteTopKByColumnGroupsBatch", "ExecuteTopKGroups", "ExecuteTopKGroupsBatch", "IndexReader", "IResearchScan", "PostingsWriter", "PreparedBatch", "Segment", "merge_gathered",
           "pred", "resolve_pred", "stage_parse_host", "sum_i128", "StreamScoredDocs", "pack_for",
           "ExecuteDistCountGroupsBatch", "ExecuteDistFacetCountsGroupsBatch", "ExecuteDistMatchAggregatesGroupsBatch",
           "MatchAggregatesDevice", "match_aggregate_device_bytes", "merge_aggregates_gathered",
           "ExecuteDistTopKByColumnGroupsBatch", "TopKByColumnDevice", "topk_by_column_device_bytes",
           "merge_topk_by_column_gathered", "ExecuteDistTopKGroupsBatch", "TopKGroupsDevice", "topk_groups_device_bytes",
           "merge_topk_groups_gathered", "ExecutePhraseCount", "ExecutePhraseCountBatch", "ExecutePhraseTopK",
           "ExecutePhraseTopKBatch", "ExecutePhraseTopKByColumn", "ExecutePhraseTopKByColumnBatch", "ExecutePhraseFacetCounts",
           "ExecutePhraseFacetCountsBatch", "ExecutePhraseMatchAggregates", "ExecutePhraseMatchAggregatesBatch",
           "ExecutePhraseMatchScan", "ExecutePhraseMatchScanBatch", "ExecutePhraseAndCount", "ExecutePhraseAndCountBatch", "ExecutePhraseAndTopK", "ExecutePhraseAndTopKBatch",
           "ExecutePhraseAndTopKByColumn", "ExecutePhraseAndTopKByColumnBatch", "ExecutePhraseAndFacetCounts", "ExecutePhraseAndFacetCountsBatch", "ExecutePhraseAndMatchAggregates", "ExecutePhraseAndMatchAggregatesBatch", "ExecutePhraseAndMatchScan", "ExecutePhraseAndMatchScanBatch",
           "ExecutePhraseGroupsCount", "ExecutePhraseGroupsCountBatch", "ExecutePhraseGroupsTopK", "ExecutePhraseGroupsTopKBatch",
           "ExecutePhraseGroupsTopKByColumn", "ExecutePhraseGroupsTopKByColumnBatch", "ExecutePhraseGroupsFacetCounts",
           "ExecutePhraseGroupsFacetCountsBatch", "ExecutePhraseGroupsMatchAggregates", "ExecutePhraseGroupsMatchAggregatesBatch",
           "ExecutePhraseGroupsMatchScan", "ExecutePhraseGroupsMatchScanBatch"]
