/*
 * oracle.h — C entry points of liboracle.so.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  This is a CPU restatement (C++17, no deps) of the algorithm of
 * TiDB's chunk-based operator hot path, written from the Go sources of pingcap/tidb as a
 * specification (the reference is pure Go and the project has no Go toolchain, so it is not
 * compiled or run: there is no oracle/_ref).  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library.  libtidbgpu.so never does.
 *
 * PARITY PINNING: the restatement is pinned against every known-answer test the reference's own
 * unit tests hold for this path (transcribed by hand in tests/test_oracle_kat.py with file:line),
 * and cross-checked against an independent nested-loop restatement of the reference's test
 * generators (inner_join_probe_test.go:80 genInnerJoinResult and siblings).  It has NOT been checked
 * against outputs of the running Go executor — "pinned by KAT, not by live reference".
 *
 * Column / chunk structs are shared with include/tidbgpu.h (same memory layout as chunk.Column).
 */
#ifndef TIDB_ORACLE_H
#define TIDB_ORACLE_H

#include "../include/tidbgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- primitives pinned by KATs ---------------------------------------------------------------- */
/* Go hash/fnv New64 (FNV-1, not 1a): used at join/row_table_builder.go:103, base_join_probe.go:297 */
uint64_t orc_fnv1_64(const uint8_t* data, size_t n);
/* join/hash_table_v2.go:55 nextPowerOfTwo (returns a power of two strictly greater than value)    */
uint64_t orc_next_power_of_two(uint64_t v);
/* join/hash_table_v2.go:67 newSubTable: table length for n valid keys                             */
uint64_t orc_hash_table_length(uint64_t valid_keys);
/* join/hash_join_v2.go:298 genHashJoinPartitionNumber / :306 getPartitionMaskOffset               */
uint32_t orc_partition_number(uint32_t concurrency);
int32_t orc_partition_mask_offset(uint32_t partition_number);
/* join/tagged_ptr.go:70 getTaggedBitsFromUintptr, :47 tagPtrHelper.init (returns taggedMask)      */
uint8_t orc_tagged_bits(uint64_t ptr);
uint64_t orc_tagged_mask(uint8_t tagged_bits);
/* codec.HashGroupKey for one int64 / float64 / NULL (util/codec/codec.go:1761): writes the encoded
 * bytes into out (cap >= 10), returns the length                                                  */
int32_t orc_group_key_int(int64_t v, int is_null, uint8_t* out);
int32_t orc_group_key_real(double v, int is_null, uint8_t* out);

/* join/join_table_meta.go:184 newTableMeta, evaluated for KATs.  Types are MySQL type codes;
 * binary_coll[i] != 0 marks a binary collation for string types.  used_in_other_cond / output_cols
 * may be NULL with n = -1 for Go nil.                                                              */
typedef struct orc_table_meta {
  int32_t key_mode;            /* 0 OneInt64, 1 FixedSerializedKey, 2 VariableSerializedKey */
  int32_t is_keys_inlined;
  int32_t is_keys_fixed_length;
  int32_t join_keys_length;
  int32_t null_map_length;
  int32_t row_length;
  int32_t is_fixed_length;
  int32_t row_data_offset;
  int32_t n_row_columns;
  int32_t row_columns_order[64];
  int32_t n_serialize_modes;
  int32_t serialize_modes[16]; /* 0 Normal, 1 NeedSignFlag, 2 KeepVarColumnLength */
  int32_t column_count_needed_for_other_condition;
} orc_table_meta;
int orc_new_table_meta(int32_t nkeys, const int32_t* build_key_index,
                       int32_t n_build_cols, const int32_t* build_types, const uint32_t* build_flags,
                       const int32_t* build_binary_coll,
                       const int32_t* build_key_types, const uint32_t* build_key_flags,
                       const int32_t* build_key_binary_coll,
                       const int32_t* probe_key_types, const uint32_t* probe_key_flags,
                       const int32_t* probe_key_binary_coll,
                       int32_t n_other, const int32_t* used_in_other_cond,
                       int32_t n_output, const int32_t* output_cols,
                       int32_t need_used_flag, orc_table_meta* out);

/* ---- hash join (HashJoinV2Exec restatement) ---------------------------------------------------- */
typedef struct orc_join orc_join;
/* concurrency = tidb_hash_join_concurrency (reference default 5, vardef/tidb_vars.go:1476,1654) */
int orc_join_open(const tg_join_desc* desc, int32_t concurrency, orc_join** out);
/* whole pipeline: build chunks -> row tables -> hash table -> probe chunks -> result, using
 * `concurrency` build and probe worker threads exactly like hash_join_v2.go:1266-1479 / :793-852 */
int orc_join_run(orc_join* j, const tg_chunk* build_chunks, int64_t n_build_chunks,
                 const tg_chunk* probe_chunks, int64_t n_probe_chunks);
/* the two phases separately: build once, probe repeatedly (bench.py's CPU baseline times the probe) */
int orc_join_build(orc_join* j, const tg_chunk* build_chunks, int64_t n_build_chunks);
int orc_join_probe(orc_join* j, const tg_chunk* probe_chunks, int64_t n_probe_chunks);
int64_t orc_join_result_rows(orc_join* j);
int32_t orc_join_result_cols(orc_join* j);
/* copy the whole result (all worker outputs concatenated) into caller buffers */
int orc_join_result_fetch(orc_join* j, tg_mut_chunk* out);
/* white-box accessors for KATs (TestKey row_table_builder_test.go:161, alignment :72)            */
int64_t orc_join_row_count(orc_join* j);
int64_t orc_join_total_row_bytes(orc_join* j);
int64_t orc_join_hash_table_slots(orc_join* j);   /* sum over partitions */
int32_t orc_join_partitions(orc_join* j);
double orc_join_build_seconds(orc_join* j);
double orc_join_probe_seconds(orc_join* j);
void orc_join_close(orc_join* j);

/* ---- hash aggregation (HashAggExec restatement) ------------------------------------------------ */
typedef struct orc_agg orc_agg;
/* partial_concurrency / final_concurrency: tidb_hashagg_partial_concurrency / final (default -1 ->
 * tidb_executor_concurrency 5, vardef/tidb_vars.go:1514-1515)                                      */
int orc_agg_open(const tg_agg_desc* desc, int32_t partial_concurrency, int32_t final_concurrency,
                 orc_agg** out);
int orc_agg_run(orc_agg* a, const tg_chunk* chunks, int64_t n_chunks);
int64_t orc_agg_result_rows(orc_agg* a);
int orc_agg_result_fetch(orc_agg* a, tg_mut_chunk* out);
double orc_agg_seconds(orc_agg* a);
void orc_agg_close(orc_agg* a);

/* ---- VecEval (row evaluator = oracle of the vector evaluator, expression/bench_test.go:1562) --- */
int orc_vec_compare_int(int op, int a_unsigned, int b_unsigned, const tg_column* a,
                        const tg_column* b, int64_t b_const, int64_t* result, uint8_t* result_nulls);
int orc_vec_compare_real(int op, const tg_column* a, const tg_column* b, double b_const,
                         int64_t* result, uint8_t* result_nulls);
int orc_vec_arith_int(int op, int a_unsigned, int b_unsigned, const tg_column* a, const tg_column* b, int64_t b_const,
                      int64_t* result, uint8_t* result_nulls);
int orc_vec_arith_real(int op, const tg_column* a, const tg_column* b, double b_const,
                       double* result, uint8_t* result_nulls);
int orc_vec_filter(const tg_chunk* chk, const tg_filter_item* items, int32_t n_items,
                   uint8_t* selected, int64_t* n_selected);

const char* orc_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
