"""universal_recommender_b200 -- H100-native Correlated Cross-Occurrence (CCO) model builder:
the train hot path of actionml/universal-recommender (URAlgorithm.calcAll -> Mahout
SimilarityAnalysis) as hand-written sm_90a CUDA behind the C ABI of include/cco_b200.h.

Host-side mirror of the reference interface for this path:
  preparator.prepare                      <- Preparator.prepare           (Preparator.scala:44-87)
  preparator.prepare_on_device            <- the same, on the GPU from string ids (cco_ingest_strings)
  IndexedDataset / BiDictionary           <- Mahout IndexedDataset
  DownsamplableCrossOccurrenceDataset     <- URAlgorithm.scala:336-340
  SimilarityAnalysis.cooccurrencesIDSs / crossOccurrenceDownsampled  <- URAlgorithm.scala:323,343
  ur_algorithm.calc_all                   <- URAlgorithm.calcAll          (URAlgorithm.scala:310-349)
  ur_algorithm.calc_all_on_device         <- calcAll through URModel.save's documents, on the GPU (cco_format_model)
  ur_algorithm.calc_pop_on_device         <- calcPop (recsModel "backfill"): an existing index re-ranked on the GPU
                                             (cco_rerank_model)
  ur_algorithm.calc_all_from_events / calc_pop_from_events  <- the same from a PredictionIO event export parsed on the
                                             GPU (cco_event_log_read: DataSource.scala:65-102); events.py is its host mirror
  ur_algorithm.user_queries_from_events / item_queries / item_set_queries  <- buildQuery for every user of an export /
                                             every item of a model index / every item set of a batch, on the GPU
                                             (cco_event_log_user_queries, cco_item_queries, cco_item_set_queries); ur_query.py
  ur_algorithm.mixed_queries_from_events  <- buildQuery for rows with any subset of {user, item, item set}, on the GPU
                                             (cco_mixed_queries); ur_query.py
  ur_algorithm.queries_from_file          <- the same for a batchpredict query file (one Query per line, each with its own
                                             template): read and rendered on the GPU (cco_query_file_*); ur_query.query_file
  ur_algorithm.index_from_pages           <- EsClient.getRDD / esJsonRDD (calcPop) and EsClient.getSource (item queries):
                                             the model index read back from Elasticsearch _search / scroll pages into the
                                             bulk body, on the GPU (cco_index_pages_*); ur_model.index_from_pages
  ur_algorithm.write_index                <- URModel.save -> EsClient.hotSwap: the mapping, bounded _bulk requests, their
                                             responses read on the GPU (cco_index_write_*), 429 retries and the alias swap,
                                             over a caller-supplied request function; ur_model.index_mapping / alias_actions
  ur_algorithm.refresh_properties_from_events / update_index  <- item properties ($set / $unset / $delete) written into
                                             the live index in place, without a retrain: the changed documents built on the
                                             GPU (cco_refresh_properties), then _bulk index and delete requests;
                                             ur_model.refresh_documents
  ur_model                                <- propertiesRDD, getRanksRDD, groupAll (URAlgorithm.scala:351-369, 537-560;
                                             URModel.scala:57-140): the host mirror of the model documents
"""
from ._native import (CcoError, CcoInvalidArgument, FLAG_ASSUME_CANONICAL, FLAG_ENTROPY_VARARGS, FLAG_KEY_RANGES, FLAG_RESULT_NO_COUNT,
                      FLAG_RESULT_NO_LLR, FLAG_ROWRATE_INTDIV, LIB_PATH)
from .events import DataSourceParams, EventWindow
from .indexed_dataset import BiDictionary, IndexedDataset
from .preparator import prepare, prepare_on_device
from .similarity_analysis import (CcoContext, CleanStats, EraseStats, DownsamplableCrossOccurrenceDataset, EventLog, IndexPages, IndexWrite, IndexWriteResult, SearchResults, SimilarityAnalysis,
                                  decode_ids, default_context, encode_ids)
from .ur_algorithm import (DefaultURAlgoParams, IndicatorParams, URAlgorithmParams, calc_all, calc_all_from_events, calc_all_on_device,
                           batchpredict_output, calc_pop_from_events, clean_export, calc_pop_on_device, index_from_pages, IndexWriteError, write_index, item_queries, item_set_queries, mixed_queries_from_events,
                           predictions_from_responses, queries_from_file, refresh_properties_from_events, refresh_properties_on_device,
                           update_index, user_queries_from_events)
from .ur_query import ItemQuery, ItemSetQuery, MixedQuery, UserQuery
from .ur_model import RankingParams, RefreshedIndex

__all__ = [
    "BiDictionary", "CcoContext", "CcoError", "CcoInvalidArgument", "DataSourceParams", "DefaultURAlgoParams", "EventWindow",
    "DownsamplableCrossOccurrenceDataset", "IndexedDataset", "IndicatorParams", "SimilarityAnalysis",
    "EventLog", "RankingParams", "URAlgorithmParams", "calc_all", "calc_all_from_events", "calc_all_on_device", "calc_pop_from_events", "clean_export", "CleanStats", "EraseStats",
    "batchpredict_output", "calc_pop_on_device", "item_queries", "item_set_queries", "mixed_queries_from_events", "predictions_from_responses", "queries_from_file", "SearchResults", "IndexPages", "index_from_pages", "IndexWrite", "IndexWriteResult", "IndexWriteError", "write_index", "refresh_properties_from_events", "refresh_properties_on_device", "update_index", "RefreshedIndex", "user_queries_from_events", "ItemQuery", "ItemSetQuery", "MixedQuery", "UserQuery", "decode_ids", "default_context", "encode_ids", "prepare", "prepare_on_device",
    "FLAG_ASSUME_CANONICAL",
    "FLAG_ENTROPY_VARARGS", "FLAG_KEY_RANGES", "FLAG_ROWRATE_INTDIV", "FLAG_RESULT_NO_COUNT", "FLAG_RESULT_NO_LLR", "LIB_PATH",
]
