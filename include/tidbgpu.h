/*
 * tidbgpu.h — C ABI of libtidbgpu.so: the H100 (sm_90a) operator hot path of TiDB's
 * chunk-based vectorized executor (hash join build/probe, hash aggregation, VecEval*
 * filter/projection kernels, key-hash repartition for multi-GPU).
 *
 * This is the drop-in boundary a cgo shim binds (see INTEGRATION.md).  TiDB has no FFI for
 * this path today; the interface it sits behind is the Go interface
 *     exec.Executor { Open(ctx) / Next(ctx, *chunk.Chunk) / Close() }
 *     (reference: pkg/executor/internal/exec/executor.go:51-77)
 * and the data that crosses it is chunk.Chunk / chunk.Column
 *     (reference: pkg/util/chunk/chunk.go:35-54, pkg/util/chunk/column.go:74-82).
 * Every entry point below names the reference function it replaces.
 *
 * Conventions
 *   - plain C, no C++ types; every call returns int: 0 = TG_OK, >0 = tg_status code.
 *     tg_last_error() returns a thread-local human readable message for the last failure.
 *   - input buffers are BORROWED for the duration of the call only (cgo pointer rule);
 *     output buffers are caller-owned and caller-sized.
 *   - a tg_join_next / tg_join_next_wait / tg_agg_next / tg_topn call that fails does not write `out` (no cell, no
 *     bitmap byte) and leaves no copy into it running: *nrows = 0, and the handle's read cursor and d2h_bytes stay
 *     where they were, so the next valid call returns the rows the failed one would have.
 *   - the library never falls back to a CPU implementation: if no CUDA device is usable every
 *     compute entry point fails with TG_ERR_CUDA.
 *   - calls on one handle are serialised internally; tg_*_close may race with an in-flight
 *     tg_*_next (executor.go:65 "Close may be called with Next at the same time"): the
 *     in-flight call returns TG_ERR_CANCELLED.
 */
#ifndef TIDBGPU_H
#define TIDBGPU_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TIDBGPU_ABI_VERSION 2

/* ---------------------------------------------------------------------------------------------
 * status codes
 * ------------------------------------------------------------------------------------------- */
typedef enum tg_status {
  TG_OK = 0,
  TG_ERR_INVALID = 1,      /* bad argument / descriptor */
  TG_ERR_UNSUPPORTED = 2,  /* valid plan, but not offloadable: the Go shim keeps the CPU executor
                              (same spirit as join.IsHashJoinV2Supported / CanUseHashJoinV2,
                              pkg/executor/builder.go:1934) */
  TG_ERR_CUDA = 3,         /* CUDA runtime failure or no device */
  TG_ERR_OOM = 4,          /* device or pinned-host allocation failed */
  TG_ERR_STATE = 5,        /* call out of order (e.g. probe before build_finish) */
  TG_ERR_CANCELLED = 6,    /* handle closed / killed while the call was running */
  TG_ERR_OVERFLOW = 7,     /* types.ErrOverflow raised by an arithmetic VecEval kernel
                              (pkg/expression/builtin_arithmetic_vec.go:513-519, :957) */
  TG_ERR_CAPACITY = 8      /* caller-provided output buffer too small */
} tg_status;

const char* tg_last_error(void);
int tg_abi_version(void);
/* number of visible CUDA devices (0 if none, never an error) */
int tg_device_count(void);
/* name / SM count / HBM bytes of a device */
int tg_device_info(int device, char* name, size_t name_cap, int* sm_count, int64_t* hbm_bytes);

/* ---------------------------------------------------------------------------------------------
 * enumerations reused verbatim from the reference so the Go shim is a plain copy
 * ------------------------------------------------------------------------------------------- */
/* pkg/parser/mysql/type.go:17-48 */
enum {
  TG_TYPE_TINY = 1, TG_TYPE_SHORT = 2, TG_TYPE_LONG = 3, TG_TYPE_FLOAT = 4, TG_TYPE_DOUBLE = 5,
  TG_TYPE_TIMESTAMP = 7, TG_TYPE_LONGLONG = 8, TG_TYPE_INT24 = 9, TG_TYPE_DATE = 10,
  TG_TYPE_DURATION = 11, TG_TYPE_DATETIME = 12, TG_TYPE_YEAR = 13, TG_TYPE_NEWDECIMAL = 0xf6,
  TG_TYPE_VARSTRING = 0xfd,
  TG_TYPE_VARCHAR = 15, TG_TYPE_BIT = 16, TG_TYPE_JSON = 0xf5, TG_TYPE_ENUM = 0xf7, TG_TYPE_SET = 0xf8,
  TG_TYPE_TINY_BLOB = 0xf9, TG_TYPE_MEDIUM_BLOB = 0xfa, TG_TYPE_LONG_BLOB = 0xfb, TG_TYPE_BLOB = 0xfc,
  TG_TYPE_STRING = 0xfe
};
/* pkg/parser/mysql/type.go:54-77 */
enum { TG_FLAG_NOT_NULL = 1u << 0, TG_FLAG_UNSIGNED = 1u << 5 };
/* pkg/planner/core/base/plan_base.go:310-322 (JoinType) */
enum {
  TG_JOIN_INNER = 0, TG_JOIN_LEFT_OUTER = 1, TG_JOIN_RIGHT_OUTER = 2, TG_JOIN_SEMI = 3,
  TG_JOIN_ANTI_SEMI = 4, TG_JOIN_LEFT_OUTER_SEMI = 5, TG_JOIN_ANTI_LEFT_OUTER_SEMI = 6
};
/* aggregate function names (pkg/parser/ast/functions.go AggFuncCount.. ) */
enum { TG_AGG_COUNT = 0, TG_AGG_SUM = 1, TG_AGG_AVG = 2, TG_AGG_MIN = 3, TG_AGG_MAX = 4,
       TG_AGG_FIRSTROW = 5 };
/* pkg/expression/aggregation/descriptor.go:155-165 (AggFunctionMode) */
enum { TG_AGGMODE_COMPLETE = 0, TG_AGGMODE_FINAL = 1, TG_AGGMODE_PARTIAL1 = 2,
       TG_AGGMODE_PARTIAL2 = 3, TG_AGGMODE_DEDUP = 4 };

/* fixed element length of a MySQL type inside a chunk column, -1 = var-len
 * (pkg/util/chunk/codec.go:165-179 getFixedLen) */
int tg_fixed_len(int mysql_type);

/* ---------------------------------------------------------------------------------------------
 * chunk.Column / chunk.Chunk views            (pkg/util/chunk/column.go:74-82, chunk.go:35-54)
 * ------------------------------------------------------------------------------------------- */
typedef struct tg_column {
  int64_t length;             /* Column.length: physical rows                                   */
  const uint8_t* null_bitmap; /* Column.nullBitmap: LSB-first, bit 1 = NOT NULL, ceil(length/8)
                                 bytes; NULL pointer = no NULLs in this column                  */
  const int64_t* offsets;     /* Column.offsets (length+1) for var-len columns, else NULL       */
  const uint8_t* data;        /* Column.data: length*elem_len little-endian bytes (fixed)       */
  int32_t elem_len;           /* 8, 4, 40, or -1 (var-len)                                      */
  int32_t reserved;
} tg_column;

typedef struct tg_chunk {
  int32_t ncols;
  int32_t reserved;
  const tg_column* cols;
  const int64_t* sel;         /* Chunk.sel: logical row i -> physical row sel[i]; NULL = identity
                                 (chunk.go:38, :394-407).  Go `int` is 64-bit on every TiDB target */
  int64_t nsel;               /* logical rows when sel != NULL (Chunk.NumRows, chunk.go:384)    */
} tg_chunk;

/* caller-owned output column: the Go side passes Column.data / Column.nullBitmap capacity */
typedef struct tg_mut_column {
  uint8_t* null_bitmap;       /* capacity ceil(capacity_rows/8) bytes, may be NULL if the caller
                                 knows the column is NOT NULL (then a NULL produced is an error) */
  uint8_t* data;              /* capacity capacity_rows*elem_len bytes                           */
  int32_t elem_len;
  int32_t reserved;
} tg_mut_column;

typedef struct tg_mut_chunk {
  int32_t ncols;
  int32_t reserved;
  tg_mut_column* cols;
  int64_t capacity_rows;
} tg_mut_chunk;

/* ---------------------------------------------------------------------------------------------
 * Chunk wire format (host code): chunk.Codec, pkg/util/chunk/codec.go — Encode :41, DecodeToChunk :93,
 * decodeColumn :101, setAllNotNull :145.  Per column: u32 length | u32 nullCount | [bitmap if nullCount > 0] |
 * [offsets (length+1) x i64 if var-len] | data.  Coprocessor / TiFlash responses use it, so a cgo shim can hand the
 * response buffer over as is (SURVEY §8 f.2).
 * ------------------------------------------------------------------------------------------- */
int tg_chunk_wire_size(const tg_chunk* chk, size_t* bytes);
int tg_chunk_encode(const tg_chunk* chk, uint8_t* buf, size_t cap, size_t* written);
/* zero copy: cols_out[i] alias buf, like the Go decoder's Columns alias the gRPC message; null_bitmap == NULL where the
 * wire carried no NULLs.  `consumed` = bytes of buf that belonged to these ncols columns.                          */
int tg_chunk_decode(const uint8_t* buf, size_t len, int32_t ncols, const int32_t* mysql_types, tg_column* cols_out,
                    size_t* consumed);
/* decode the fixed-width columns straight into caller-owned (e.g. tg_host_alloc'ed, pinned) buffers; columns whose
 * out->cols[i].data is NULL are skipped                                                                           */
int tg_chunk_decode_into(const uint8_t* buf, size_t len, int32_t ncols, const int32_t* mysql_types, tg_mut_chunk* out,
                         int64_t* rows, size_t* consumed);

/* ---------------------------------------------------------------------------------------------
 * pinned host memory for a chunk.ColumnAllocator (pkg/util/chunk/column.go:85) backed by
 * cudaHostAlloc, precedent: pkg/lightning/manual/manual.go (C.calloc behind Go slices).
 * Buffers from here make H2D/D2H copies true DMA; any other host pointer is accepted too.
 * ------------------------------------------------------------------------------------------- */
int tg_host_alloc(size_t bytes, void** out);
int tg_host_free(void* p);

/* raw device memory + copies, for device-resident ("synthetic columnar") runs and tests */
int tg_dev_alloc(int device, size_t bytes, void** out);
int tg_dev_free(int device, void* p);
int tg_memcpy_h2d(int device, void* dst_dev, const void* src_host, size_t bytes);
int tg_memcpy_d2h(int device, void* dst_host, const void* src_dev, size_t bytes);
/* Asynchronous device-to-device copy on `stream` (cudaMemcpyAsync, copy engine): `dst` may be memory of a peer GPU mapped
 * with tg_ipc_open — the DMA then crosses NVLink without occupying SMs (SegmentExchange's transfer step).          */
int tg_memcpy_d2d_async(int device, void* dst_dev, const void* src_dev, size_t bytes, void* stream);
int tg_device_synchronize(int device);

/* ---------------------------------------------------------------------------------------------
 * Hash join                      replaces join.HashJoinV2Exec (pkg/executor/join/hash_join_v2.go:608)
 * ------------------------------------------------------------------------------------------- */
typedef struct tg_join tg_join;

/* scalar filter program: CNF of (column OP constant) / (column OP column) items on 8-byte columns;
 * replaces expression.VectorizedFilter (pkg/expression/chunk_executor.go:413) for
 * BuildFilter / ProbeFilter / OtherCondition (pkg/executor/builder.go:1771-1931). */
enum { TG_CMP_LT = 0, TG_CMP_LE = 1, TG_CMP_GT = 2, TG_CMP_GE = 3, TG_CMP_EQ = 4, TG_CMP_NE = 5 };
typedef struct tg_filter_item {
  int32_t op;          /* TG_CMP_*                                                      */
  int32_t lhs_col;     /* column index in the chunk the filter is evaluated on           */
  int32_t rhs_col;     /* -1 = compare with constant                                     */
  int32_t is_real;     /* 0: int64 compare (signed unless lhs_unsigned), 1: float64      */
  int32_t lhs_unsigned;
  int32_t rhs_unsigned; /* signedness of the right column / constant (types.CompareInt takes both flags) */
  int64_t const_i64;   /* constant when rhs_col < 0 and !is_real                         */
  double const_f64;    /* constant when rhs_col < 0 and is_real                          */
} tg_filter_item;

/* One CNF item of HashJoinV2Exec.OtherCondition (inner_join_probe.go:72-79, base_join_probe.go:758
 * buildResultAfterOtherCondition): `operand OP operand` over the JOINED row, each operand a column of the left or the
 * right child (side 0 / 1), the right operand optionally a constant (rhs_side = -1).  A candidate pair (equal keys)
 * is a match only if every item is non-NULL true (VectorizedFilter semantics).                                     */
typedef struct tg_other_item {
  int32_t op;            /* TG_CMP_*                                                      */
  int32_t is_real;       /* 0: int64 compare, 1: float64                                  */
  int32_t lhs_side, lhs_col;
  int32_t rhs_side, rhs_col;   /* rhs_side = -1: constant                                 */
  int32_t lhs_unsigned, rhs_unsigned;
  int64_t const_i64;
  double const_f64;
} tg_other_item;

typedef struct tg_join_desc {
  int32_t join_type;          /* TG_JOIN_*                                                       */
  int32_t build_is_right;     /* HashJoinV2Exec RightAsBuildSide: 1 = right child is build side  */
  /* schema of both children: MySQL type + flag per column (FieldType.tp / .flag)               */
  int32_t n_left_cols;
  int32_t n_right_cols;
  const int32_t* left_types;  const uint32_t* left_flags;
  const int32_t* right_types; const uint32_t* right_flags;
  /* equal-condition keys: column index per side (BuildKeyColIdx / ProbeKeyColIdx after
   * mapping to left/right, builder.go:1780-1830).  nkeys = 1: int family / float / double key (OneInt64 mode and the
   * 8-byte fixed keys).  nkeys = 2..4: FixedSerializedKey mode (join_table_meta.go:174-178) for 8-byte integer-family
   * columns — a row with a NULL in any key column has no key; a pair matches iff every key column is equal by value
   * (signed vs unsigned compared by value).  Join shapes that need a build-side scan or the NULL-aware match flag are
   * declined with several keys (TG_ERR_UNSUPPORTED → the planner keeps the CPU executor), like with OtherCondition.  */
  int32_t nkeys;
  int32_t reserved0;
  const int32_t* left_key_idx;
  const int32_t* right_key_idx;
  /* output = LUsed columns of left ‖ RUsed columns of right (builder.go:1868-1871).
   * NULL pointer with n = -1 means "all columns" (the reference's nil slice).  Used columns may be 4/8-byte fixed-width
   * columns or DECIMAL (TG_TYPE_NEWDECIMAL, 40-byte MyDecimal cells) on either side, for every join type: a DECIMAL cell
   * is moved as its 40 raw bytes, never interpreted, so a non-NULL output cell is bit-identical to its input cell
   * (non-canonical forms, resultFrac and unused words included) and a cell under NULL is zero bytes.  No key, filter
   * item or OtherCondition operand may be a DECIMAL column (TG_ERR_UNSUPPORTED).                                    */
  int32_t n_lused; int32_t n_rused;
  const int32_t* lused; const int32_t* rused;
  /* optional filters evaluated on the build-side / probe-side child chunk                      */
  int32_t n_build_filter; int32_t n_probe_filter;
  const tg_filter_item* build_filter;
  const tg_filter_item* probe_filter;
  int32_t device;             /* CUDA device ordinal                                             */
  int32_t reserved1;
  void* stream;               /* cudaStream_t to launch on; NULL = library-owned stream          */
  double load_factor;         /* 0 = default                                                     */
  /* OtherCondition (non-equi residual evaluated on candidate pairs); offloaded for inner, probe-side outer, semi and
   * anti-semi joins with the right child as build side (the gate declines the rest)              */
  int32_t n_other_cond; int32_t reserved2;
  const tg_other_item* other_cond;
} tg_join_desc;

/* planner gate: 0 if this descriptor can run on the GPU, TG_ERR_UNSUPPORTED otherwise        */
int tg_join_supported(const tg_join_desc* desc);

/* HashJoinV2Exec.Open (hash_join_v2.go:690)                                                  */
int tg_join_open(const tg_join_desc* desc, tg_join** out);
/* buildWorkerBase.fetchBuildSideRows + BuildWorkerV2.processOneChunk (hash_join_base.go:257,
 * hash_join_v2.go:536): one build-side child chunk. Host buffers; copied before returning.    */
int tg_join_build_push(tg_join* j, const tg_chunk* chk);
/* same, columns already resident in device memory (borrowed until tg_join_build_finish)       */
int tg_join_build_push_dev(tg_join* j, const tg_chunk* dev_chk);
/* mergeRowTablesToHashTable + buildHashTable (hash_join_v2.go:217, :1458)                     */
int tg_join_build_finish(tg_join* j);
/* ProbeWorkerV2.processOneProbeChunk → JoinProbe.SetChunkForProbe + Probe
 * (hash_join_v2.go:932, base_join_probe.go:179, inner_join_probe.go:27): one probe-side child
 * chunk from host memory.  The library batches internally; joined rows become available to
 * tg_join_next.                                                                               */
int tg_join_probe_push(tg_join* j, const tg_chunk* chk);
/* end of probe side: flush the batcher; for build-side-outer joins also runs
 * JoinProbe.ScanRowTable (outer_join_probe.go:117)                                            */
int tg_join_probe_finish(tg_join* j);
/* HashJoinV2Exec.Next (hash_join_v2.go:1161): fill at most min(max_rows, out->capacity_rows)
 * joined rows; *nrows == 0 means EOF (only after tg_join_probe_finish).                       */
int tg_join_next(tg_join* j, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows);
/* Same, but blocks until rows are available or the probe side is finished (then 0 = EOF).  One thread may sit in
 * tg_join_next_wait while another pushes probe chunks — the reference's probe fetcher goroutine vs the consumer of
 * joinResultCh (hash_join_v2.go:840, :1176); results are copied on their own stream, so D2H overlaps the next H2D. */
int tg_join_next_wait(tg_join* j, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows);
/* Start another probe pass against the SAME built table (results not yet fetched are dropped).  Mirrors re-execution
 * of the probe side under Apply with a cached build side; not available for joins that scan the build side. */
int tg_join_probe_rewind(tg_join* j);
/* HashJoinV2Exec.Close (hash_join_v2.go:647); idempotent                                     */
int tg_join_close(tg_join* j);

/* Device-resident probe (inputs and outputs stay in HBM): probe `dev_chk` against the built table,
 * write the joined columns into library-owned device buffers, return their device pointers.
 * out_cols[i] receives the device address of output column i (n_lused+n_rused entries),
 * out_nulls[i] the device null bitmap of that column or NULL.  Valid until the next probe call
 * on this handle or close.  This is the kernel-only path bench.py times as `value`.           */
int tg_join_probe_dev(tg_join* j, const tg_chunk* dev_chk, int64_t* out_rows,
                      void** out_cols, void** out_nulls);
/* Same, for a device chunk that is SEGMENTED: `nseg` segments of `seg_cap` rows each (seg_cap a multiple of
 * 1024), segment s holding seg_cnt_dev[s] valid rows at its start; dev_chk->cols[*].length = nseg*seg_cap.  This is
 * the shape a count-free exchange delivers (tg_partition_exchange_cf: one fixed-capacity region per sending GPU,
 * fill counts known only on the device), so the receiver probes without compacting and without a host round trip.
 * Only for plans the fused fast path covers (tg_join_get_stats().table_mode == 1); others: TG_ERR_UNSUPPORTED.
 * DECIMAL probe and build output columns are accepted: the fused kernels carry them as row ids, as on the other paths. */
int tg_join_probe_dev_seg(tg_join* j, const tg_chunk* dev_chk, const int64_t* seg_cnt_dev, int32_t nseg,
                          int64_t seg_cap, int64_t* out_rows, void** out_cols, void** out_nulls);


/* hashJoinRuntimeStatsV2 (pkg/executor/join/hash_join_stats.go:142)                          */
typedef struct tg_join_stats {
  int64_t build_rows;         /* rows pushed on the build side                       */
  int64_t build_valid_keys;   /* rows inserted into the table (non-NULL key, passed filter) */
  int64_t table_slots;        /* slots allocated                                      */
  int64_t distinct_keys;
  int64_t max_dup;            /* largest multiplicity of one key                      */
  int64_t probe_rows;
  int64_t output_rows;
  int64_t kernel_launches;    /* CUDA kernels launched by this handle                 */
  int32_t table_mode;         /* 0 none, 1 unique-inline, 2 grouped row store         */
  int32_t paths;              /* TG_JOIN_PATH_* bits: kernel families this handle has launched */
  double build_ms, probe_ms;  /* device time measured with CUDA events                */
  int64_t h2d_bytes, d2h_bytes;
} tg_join_stats;
/* tg_join_stats.paths */
enum {
  TG_JOIN_PATH_PROBE_UQ = 1 << 0,       /* single-pass unique-key probe (k_probe_inner_uq)                       */
  TG_JOIN_PATH_PROBE_GENERAL = 1 << 1,  /* general count -> scan -> write probe                                  */
  TG_JOIN_PATH_PROBE_DIRECT = 1 << 2,   /* fused warp probe (k_probe_inner_u1_w), also the gated fallback launch  */
  TG_JOIN_PATH_PROBE_SEG = 1 << 3,      /* segment probe over L2-partitioned rows (k_probe_inner_u1_seg_lean)    */
  /* 1 << 4 is unassigned: older headers name a removed kernel with it, so a new path must not reuse it              */
  TG_JOIN_PATH_SCATTER_BULK = 1 << 5,   /* bulk partition scatter (k_partition_scatter_bulk)                     */
  TG_JOIN_PATH_SCATTER = 1 << 6,        /* LSU partition scatter over the whole input (k_partition_scatter)      */
  TG_JOIN_PATH_CELL_GATHER = 0x80,      /* 1 << 7: DECIMAL output cells gathered from row ids (k_gather_cells)      */
  TG_JOIN_PATH_PROBE_INDEX = 0x100,     /* 1 << 8: in-place segment probe through the table's slice index
                                           (k_probe_inner_u1_seg_inplace_pidx)                                        */
  TG_JOIN_SCATTER_TILE_4K = 0x200       /* 1 << 9, not a kernel family but a qualifier of TG_JOIN_PATH_SCATTER_BULK: the
                                           bulk scatter ran with 4096-row tiles (dense input), else with 1024-row tiles   */
};
int tg_join_get_stats(tg_join* j, tg_join_stats* out);

/* ---------------------------------------------------------------------------------------------
 * Hash aggregation            replaces aggregate.HashAggExec (pkg/executor/aggregate/agg_hash_executor.go:93)
 * ------------------------------------------------------------------------------------------- */
typedef struct tg_agg tg_agg;

typedef struct tg_agg_func {
  int32_t name;      /* TG_AGG_*                                                               */
  int32_t mode;      /* TG_AGGMODE_*                                                           */
  int32_t arg_col;   /* input column index; -1 for COUNT(*) / count(constant)                  */
  int32_t arg_type;  /* MySQL type of the argument (TG_TYPE_DOUBLE / TG_TYPE_LONGLONG ...)      */
  uint32_t arg_flag;
  int32_t arg_col2;  /* Final/Partial2 AVG: second input column (count, then sum: func_avg.go:444);
                      * arg_expr != 0: the second column of the argument expression                */
  /* The argument as a small scalar expression instead of a plain column (AggFuncDesc.Args[0] is an expression.Expression
   * evaluated per row: args[0].EvalReal, func_sum.go:90).  Fused into the update kernel — no projected column is
   * materialised.  DOUBLE columns, SUM / AVG in Complete mode.  NULL if either column is NULL; a non-finite intermediate
   * on a non-NULL row fails the call with TG_ERR_OVERFLOW (builtinArithmetic{Minus,Multiply}RealSig).
   *   TG_ARGEXPR_COL        arg_col
   *   TG_ARGEXPR_MUL        arg_col * arg_col2
   *   TG_ARGEXPR_MUL_CSUB   arg_col * (arg_const - arg_col2)      e.g. l_extendedprice * (1 - l_discount)            */
  int32_t arg_expr;
  /* AggFuncDesc.RetTp: GetType() and GetDecimal().  Any ret_type other than TG_TYPE_NEWDECIMAL (0 = not given) keeps the
   * result type the function has always had here.  TG_TYPE_NEWDECIMAL asks for TiDB's exact DECIMAL result of SUM / AVG
   * over an integer column (typeInfer4Sum / typeInfer4Avg, aggregation/base_func.go; the shim unwraps the
   * cast(col AS DECIMAL) that WrapCastForAggArgs puts around it):
   *   - Complete mode, arg_expr = TG_ARGEXPR_COL, an 8-byte integer-family column, signed or TG_FLAG_UNSIGNED;
   *     anything else is TG_ERR_UNSUPPORTED.  SUM needs ret_frac = 0 and AVG 0 <= ret_frac <= 30, else TG_ERR_INVALID.
   *   - SUM is the exact sum (NULL when the group has no non-NULL input, func_sum.go sum4Decimal).  AVG is
   *     DecimalDiv(sum, count, ret_frac) rounded to ret_frac digits with ModeHalfUp (func_avg.go baseAvgDecimal): the
   *     quotient is truncated at 9 * ceil(ret_frac / 9) fraction digits, so AVG rounds half away from zero unless ret_frac
   *     is a multiple of 9, where it truncates toward zero.  NULL when the count is 0.  A result that is zero is never
   *     negative.
   *   - The output column holds 40-byte MyDecimal cells (types/mydecimal.go MyDecimal, copied whole into a chunk column):
   *     int8 digitsInt, int8 digitsFrac, int8 resultFrac, bool negative, int32 wordBuf[9] in base 10^9, most significant
   *     word first, integer words then fraction words, unused words 0.  The library writes one canonical form:
   *     digitsInt = 9 * the number of integer words (at least one word, as FromUint makes it), digitsFrac = resultFrac =
   *     ret_frac.  tg_agg_next fails with TG_ERR_INVALID unless the caller's tg_mut_column.elem_len for that column is 40;
   *     tg_agg_result_dev returns a device column of 40-byte cells.
   *   - SUM / AVG / MIN / MAX over a DECIMAL column follow the same rules at the column's scale: see tg_agg_desc_ex.
   * The table keeps such a function in three 8-byte words (128-bit sum lo / hi, non-NULL count), so a plan needs at most
   * 24 state words in all; more is TG_ERR_UNSUPPORTED.                                                                     */
  int16_t ret_type;
  int16_t ret_frac;
  double arg_const;
} tg_agg_func;
enum { TG_ARGEXPR_COL = 0, TG_ARGEXPR_MUL = 1, TG_ARGEXPR_MUL_CSUB = 2 };

typedef struct tg_agg_desc {
  int32_t n_cols;                 /* child schema                                               */
  int32_t n_group_by;
  const int32_t* col_types; const uint32_t* col_flags;
  const int32_t* group_by_cols;   /* GroupByItems as plain column refs (agg_util.go:106)        */
  int32_t n_funcs;
  int32_t device;
  const tg_agg_func* funcs;       /* AggFuncDescs (builder.go:2106-2181)                        */
  void* stream;
  int64_t expected_groups;        /* hint (planner NDV estimate); 0 = grow on demand            */
} tg_agg_desc;

/* tg_agg_desc plus the precision and scale of the child columns, for aggregates over DECIMAL(p <= 18) columns.
 * tg_agg_supported / tg_agg_open are tg_agg_supported_ex / tg_agg_open_ex with both arrays NULL.
 *   col_flen[c]    = FieldType.GetFlen() of child column c, col_decimal[c] = FieldType.GetDecimal(); NULL or -1 = not given.
 * A function whose argument column is TG_TYPE_NEWDECIMAL is offloaded when the mode is Complete, arg_expr is
 * TG_ARGEXPR_COL, 1 <= flen <= 18 and 0 <= decimal <= flen, and (s = the column's decimal):
 *   SUM    ret_type TG_TYPE_NEWDECIMAL, ret_frac = s: the exact sum at scale s (typeInfer4Sum, aggregation/base_func.go;
 *          sum4Decimal, func_sum.go)
 *   AVG    ret_type TG_TYPE_NEWDECIMAL, s <= ret_frac <= 30: DecimalDiv(sum, count) rounded to ret_frac digits with
 *          ModeHalfUp, by the truncate-then-round rule of tg_agg_func.ret_type (typeInfer4Avg; avgOriginal4Decimal /
 *          baseAvgDecimal, func_avg.go)
 *   MIN / MAX  ret_type TG_TYPE_NEWDECIMAL, ret_frac = s: the smallest / largest value, at scale s (typeInfer4MaxMin;
 *          max4Decimal / min4Decimal, func_max_min.go:906)
 *   COUNT  its usual BIGINT result (only the null bitmap is read)
 * A scale rule not met or decimal > flen is TG_ERR_INVALID.  flen > 18, flen / decimal not given, Final / Partial2 mode
 * (a partial DECIMAL sum has p + 22 digits), FIRSTROW, a DECIMAL GROUP BY column or a non-DECIMAL ret_type over a
 * DECIMAL argument is TG_ERR_UNSUPPORTED.  SUM / AVG keep the 128-bit sum of tg_agg_func.ret_type (2-3 state words),
 * MIN / MAX 1-2 words, under the same 24-word limit.
 * SUM / AVG of a product, arg_expr TG_ARGEXPR_MUL (arg_col * arg_col2) or TG_ARGEXPR_MUL_CSUB (arg_col * (c - arg_col2),
 * c = arg_const), are offloaded when both columns are DECIMAL with 1 <= flen <= 18 and 0 <= decimal <= flen (the same
 * column may be both), the mode is Complete, ret_type is TG_TYPE_NEWDECIMAL and s = s_a + s_b <= 30; for MUL_CSUB c must be
 * a finite integer with |c| * 10^s_b <= 10^18.  The value is the exact product (DecimalMul; c - b is exact at scale s_b)
 * at scale s.  SUM needs ret_frac = s, AVG s <= ret_frac <= 30 (TG_ERR_INVALID otherwise); results follow the column rules
 * above at scale s.  s > 30, a constant that is not such an integer, a DECIMAL operand paired with a DOUBLE or integer one,
 * flen > 18, MIN / MAX / COUNT of an expression and Final / Partial modes are TG_ERR_UNSUPPORTED.  The state is an exact
 * 192-bit sum (3 words, 4 with a nullable operand), under the same 24-word limit.
 * Input columns hold 40-byte MyDecimal cells (elem_len 40, host or device memory; device columns need only 8-byte
 * alignment).  A non-NULL cell must be in the column's stored form, as MyDecimal.FromBin (types/mydecimal.go:1465) makes
 * it: digitsFrac = decimal, ceil(digitsInt / 9) integer words (digitsInt may be 0, leading words may be 0), then
 * ceil(decimal / 9) fraction words, left-aligned (0.5 at decimal 1 is the word 500000000), at most flen significant
 * digits; resultFrac is ignored and a negative zero is 0.  A push with any other non-NULL cell fails with TG_ERR_INVALID
 * and leaves the groups unchanged.  Cells under NULL are not looked at.  Results are cells in the canonical form of
 * tg_agg_func.ret_type, with digitsFrac = resultFrac = ret_frac.                                                      */
typedef struct tg_agg_desc_ex {
  tg_agg_desc base;               /* first member: everything tg_agg_desc says, unchanged       */
  const int32_t* col_flen;        /* FieldType.GetFlen() per child column; NULL = not given      */
  const int32_t* col_decimal;     /* FieldType.GetDecimal() per child column; NULL = not given   */
} tg_agg_desc_ex;

/* tg_agg_desc_ex plus AggFuncDesc.HasDistinct per function, for COUNT, SUM and AVG with DISTINCT in Complete mode
 * (aggfuncs/builder.go: countOriginalWithDistinct*, sum4Distinct*, avgOriginal4Distinct*).  has_distinct NULL or all 0:
 * tg_agg_supported_ex2 / tg_agg_open_ex2 answer exactly like tg_agg_supported_ex / tg_agg_open_ex.
 * A DISTINCT function aggregates each distinct non-NULL value of its argument once per group.  Groups are formed as
 * without DISTINCT (NULL keys make one group, a DOUBLE key -0 is +0), and a value seen in an earlier push of the handle
 * stays seen.  Values are distinct by:
 *   integer family (signed, TG_FLAG_UNSIGNED, YEAR, DURATION)   the 64 bits (Int64Set)
 *   DOUBLE                                                      -0 and +0 are one value; every NaN row is a new value
 *                                                               (Go map[float64]: NaN != NaN)
 *   DECIMAL(flen <= 18, decimal)                                the value at the column's scale (MyDecimal.ToHashKey:
 *                                                               1.50 = 1.5)
 *   COUNT(DISTINCT x)   BIGINT, the number of distinct values; 0 for a group without one
 *   SUM(DISTINCT x)     the sum of the distinct values, NULL without one
 *   AVG(DISTINCT x)     that sum divided by the number of distinct values; a DECIMAL result is rounded by the rule of
 *                       tg_agg_func.ret_type
 *   MIN / MAX           HasDistinct changes nothing (buildMaxMin ignores it)
 * Without GROUP BY, empty input gives the usual default row (COUNT 0, SUM and AVG NULL).  A DISTINCT function is
 * accepted when the same function without DISTINCT is (same argument types, ret_type / ret_frac rules and 24-word
 * limit; COUNT over a DECIMAL(flen <= 18) column included), and it needs a free column slot: child columns plus distinct
 * DISTINCT argument columns <= 16.  TG_ERR_UNSUPPORTED: DISTINCT in Final / Partial modes, an argument expression
 * (arg_expr != TG_ARGEXPR_COL), a date-time, string, FLOAT or DECIMAL(flen > 18) argument, COUNT(DISTINCT a, b)
 * (arg_col2 >= 0: arg_col2 must be -1) and FIRSTROW.  DISTINCT with arg_col < 0 is TG_ERR_INVALID.
 * The library keeps one dedup set per DISTINCT argument column, in device memory, for the life of the handle; COUNT,
 * SUM and AVG with DISTINCT over one column share it.  It grows on demand; a push whose growth cannot be allocated fails
 * with TG_ERR_OOM, and every later push and finish of that handle fails with TG_ERR_STATE (the set already holds
 * values of rows that were not aggregated).  A push that fails on a bad DECIMAL cell leaves groups and sets unchanged. */
typedef struct tg_agg_desc_ex2 {
  tg_agg_desc_ex ex;              /* everything tg_agg_desc_ex says, unchanged                  */
  const uint8_t* has_distinct;    /* AggFuncDesc.HasDistinct per function (n_funcs); NULL = none */
} tg_agg_desc_ex2;

int tg_agg_supported(const tg_agg_desc* desc);
int tg_agg_supported_ex(const tg_agg_desc_ex* desc);
int tg_agg_supported_ex2(const tg_agg_desc_ex2* desc);
/* HashAggExec.Open (agg_hash_executor.go:237) */
int tg_agg_open(const tg_agg_desc* desc, tg_agg** out);
int tg_agg_open_ex(const tg_agg_desc_ex* desc, tg_agg** out);
int tg_agg_open_ex2(const tg_agg_desc_ex2* desc, tg_agg** out);
/* fetchChildData + HashAggPartialWorker.updatePartialResult (agg_hash_executor.go:449,
 * agg_hash_partial_worker.go:256): one child chunk (host / device-resident)                    */
int tg_agg_push(tg_agg* a, const tg_chunk* chk);
int tg_agg_push_dev(tg_agg* a, const tg_chunk* dev_chk);
/* end of input: HashAggFinalWorker merge + result generation (agg_hash_final_worker.go:73,:121) */
int tg_agg_finish(tg_agg* a);
/* HashAggExec.Next (agg_hash_executor.go:441). Output schema = one column per agg func in
 * desc order (the reference emits group columns through firstrow() funcs, SURVEY §8 note 4).
 * Each output column's elem_len must be its result's width (40 for a DECIMAL result, else 8) and a column that can be
 * NULL needs a null_bitmap; otherwise TG_ERR_INVALID, with nothing written.                       */
int tg_agg_next(tg_agg* a, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows);
int tg_agg_close(tg_agg* a);
/* device-resident result: number of groups + device pointers of the output columns            */
int tg_agg_result_dev(tg_agg* a, int64_t* out_rows, void** out_cols, void** out_nulls);

typedef struct tg_agg_stats {
  int64_t input_rows, groups, table_slots, kernel_launches;
  double update_ms, finalize_ms;
  int64_t h2d_bytes, d2h_bytes;
  int64_t local_rows;         /* rows the CTA-local (shared-memory) level of the grouped update absorbed       */
  int32_t paths;              /* TG_AGG_PATH_* bits: kernel families this handle has launched                 */
  int32_t reserved;
} tg_agg_stats;
/* tg_agg_stats.paths */
enum {
  TG_AGG_PATH_NOGROUP = 1 << 0,     /* no GROUP BY (k_agg_update_nogroup)                                        */
  TG_AGG_PATH_V2_GLOBAL = 1 << 1,   /* grouped update, global table only (k_agg_update2<false>)                 */
  TG_AGG_PATH_V2_LOCAL = 1 << 2,    /* grouped update with the CTA-local level (k_agg_update2<true>)            */
  TG_AGG_PATH_MULTI_KEY = 1 << 3,   /* several GROUP BY columns (k_agg_update_mk)                                */
  TG_AGG_PATH_V1_LOCAL = 1 << 4,    /* TG_AGG_V1=1: CTA-local partial pass (k_agg_update_local)                  */
  TG_AGG_PATH_V1_GLOBAL = 1 << 5,   /* TG_AGG_V1=1: global update (k_agg_update)                                 */
  TG_AGG_PATH_MERGE = 1 << 6        /* partial results folded into the global table (k_agg_merge)                */
};
int tg_agg_get_stats(tg_agg* a, tg_agg_stats* out);
/* the dedup pass of the DISTINCT functions (k_agg_distinct_mark), cumulative over the handle's pushes: (group, value)
 * pairs in the sets (NaN rows never enter one), slots of all sets, set growths, mark kernel launches, and the device time
 * of the pass including its growth (CUDA events).  All 0 for a plan without DISTINCT. */
typedef struct tg_agg_distinct_stats {
  int64_t pairs, set_slots, set_grows, launches;
  double mark_ms;
} tg_agg_distinct_stats;
int tg_agg_get_distinct_stats(tg_agg* a, tg_agg_distinct_stats* out);

/* tg_agg_desc_ex2 plus FieldType.GetCollate() (a MySQL collation id) per child column, for GROUP BY over string columns.
 * col_collation NULL, or a plan without a string column: tg_agg_supported_ex3 / tg_agg_open_ex3 answer exactly like
 * tg_agg_supported_ex2 / tg_agg_open_ex2.
 *   String column: col_types TG_TYPE_VARCHAR, TG_TYPE_VARSTRING, TG_TYPE_STRING or one of the four BLOB / TEXT types
 *     (ENUM, SET, JSON and BIT are TG_ERR_UNSUPPORTED wherever they are used).
 *   GROUP BY: a string GROUP BY column needs col_collation 63 (binary), 46 (utf8mb4_bin), 83 (utf8_bin), 65 (ascii_bin),
 *     47 (latin1_bin) or 309 (utf8mb4_0900_bin); any other id is TG_ERR_UNSUPPORTED.  The group key is
 *     collator.ImmutableKey (codec.go HashGroupKey): the bytes under 63 and 309, the bytes with trailing 0x20 cut under
 *     46, 83, 65 and 47 ("a", "a " and "a  " form one group, "a\t" its own).  NULL is its own group, apart from ''.  Keys
 *     are equal only when their key bytes are.  String columns count toward the 4 GROUP BY columns and mix with integer
 *     and DOUBLE ones.
 *   Functions over a string column: FIRSTROW of a string GROUP BY column, and COUNT without DISTINCT (only the NULL
 *     bitmap is read).  SUM, AVG, MIN, MAX, any DISTINCT function and a string operand of arg_expr are
 *     TG_ERR_UNSUPPORTED.  FIRSTROW of a string GROUP BY column returns the raw bytes, trailing spaces included, of the
 *     group's earliest row in push order (within a chunk, logical row order: `sel` order when it has one), as
 *     firstRow4String with one worker (aggfuncs/func_first_row.go); NULL for the NULL group.  Under 46, 83, 65 and 47
 *     with several GROUP BY columns, rows of one key value in different groups may differ in their trailing spaces, so
 *     such a FIRSTROW also takes, per key column, one free column slot (child columns + DISTINCT argument columns +
 *     such columns <= 16) and one of the 12 aggregate slots and one state word (a per-group MIN the library adds and
 *     does not return); a plan past those limits is TG_ERR_UNSUPPORTED.  A push to such a plan fails with
 *     TG_ERR_UNSUPPORTED when a row of that column has 2^23 or more trailing spaces, or when the handle's input would
 *     reach 2^41 rows.  FIRSTROW of a string column that is not a GROUP BY column stays TG_ERR_UNSUPPORTED.
 *   Pushes: a string column has elem_len -1 and length + 1 offsets, under the Columns and Offsets rules of
 *     tg_vec_filter_ex2 (offsets need not start at 0; a bad row is TG_ERR_INVALID).  A host push checks the offsets of
 *     every row it holds before it stages anything; a device push (offsets 8-byte aligned) checks every row on the
 *     device before the dictionaries see the batch.  A rejected push leaves groups, DISTINCT sets and dictionaries
 *     unchanged.  A push that fails once a dictionary has run its encode pass on the batch (an allocation failure while
 *     a dictionary or the group table grows, a too-wide trailing-space count above) fails with its status, and every
 *     later push and finish fails with TG_ERR_STATE.  A failure before that pass (a bad row, an allocation before the
 *     first round) leaves the handle usable.
 *   Results: a string result column (FIRSTROW of a string column) is read with tg_agg_next_ex or tg_agg_result_dev_ex;
 *     tg_agg_next and tg_agg_result_dev return TG_ERR_INVALID for such a plan and write nothing.
 * The library keeps one device dictionary per string GROUP BY column for the life of the handle: an id per key value,
 * the raw bytes of its earliest row, and a hash table that grows on demand (tg_agg_get_string_stats). */
typedef struct tg_agg_desc_ex3 {
  tg_agg_desc_ex2 ex2;            /* everything tg_agg_desc_ex2 says, unchanged                  */
  const int32_t* col_collation;   /* FieldType.GetCollate() per child column; NULL = not given   */
} tg_agg_desc_ex3;
int tg_agg_supported_ex3(const tg_agg_desc_ex3* desc);
int tg_agg_open_ex3(const tg_agg_desc_ex3* desc, tg_agg** out);

/* A caller-owned var-length result column: offsets has room for capacity_rows + 1 values, data for data_cap bytes. */
typedef struct tg_mut_varlen { int64_t* offsets; uint8_t* data; int64_t data_cap; } tg_mut_varlen;
/* tg_agg_next with string results.  var_out has one entry per result column; only the string ones are read (their
 * tg_mut_column has elem_len -1 and its data pointer is ignored; its null_bitmap follows the usual rules).  Serves the
 * largest n <= min(max_rows, capacity_rows, rows left) whose bytes fit data_cap in every string column, and writes
 * offsets[0..n] from 0 and the bytes.  If not even one row fits: TG_ERR_CAPACITY, nothing written, the read position
 * unchanged.  For a plan without string results it is tg_agg_next, and var_out may be NULL. */
int tg_agg_next_ex(tg_agg* a, tg_mut_chunk* out, tg_mut_varlen* var_out, int64_t max_rows, int64_t* nrows);
/* tg_agg_result_dev plus out_offsets: for a string result, out_cols[k] is its device bytes and out_offsets[k] its device
 * offsets (rows + 1 int64 values from 0); NULL for every other result. */
int tg_agg_result_dev_ex(tg_agg* a, int64_t* out_rows, void** out_cols, void** out_nulls, void** out_offsets);

/* the encode pass of the string GROUP BY columns (k_str_dict_encode), cumulative over the handle: dictionary entries,
 * arena bytes and table slots of all dictionaries, table growths, kernel launches of the pass (growth and arena copies
 * included), and its device time (CUDA events).  All 0 for a plan without a string GROUP BY column. */
typedef struct tg_agg_string_stats {
  int64_t dict_entries, dict_bytes, dict_slots, dict_grows, launches;
  double encode_ms;
} tg_agg_string_stats;
int tg_agg_get_string_stats(tg_agg* a, tg_agg_string_stats* out);
/* tg_agg_stats.paths bit 7 (0x80): the encode pass of a string GROUP BY column ran (k_str_dict_encode) */
enum { TG_AGG_PATH_STRING_KEY = 0x80 };

/* ---------------------------------------------------------------------------------------------
 * VecEval* kernels             replace pkg/expression builtin_*_vec.go signatures
 * All operate on one column-at-a-time over host or device buffers (`on_device` flag).
 * Result null bitmap = MergeNulls of the argument bitmaps (pkg/util/chunk/column.go:906).
 * Every call below checks its arguments (descriptors, types, elem_len, alignment, items, constants, collations, host
 * offsets bounds) before it looks for the device: a bad argument gets the same status on a machine without a device.
 * A failed call with host buffers (on_device == 0) writes nothing: no result value, no bitmap byte, no `selected` byte,
 * and *n_selected is left unset.  With device buffers, `result` / `result_nulls` / `selected` may have been written;
 * *n_selected is not.
 * ------------------------------------------------------------------------------------------- */
enum { TG_ARITH_PLUS = 0, TG_ARITH_MINUS = 1, TG_ARITH_MUL = 2 };

/* builtinLTIntSig.vecEvalInt & friends (pkg/expression/builtin_compare_vec.go:524-561, :619):
 * result int64 0/1, NULL if either side NULL.  b == NULL -> compare with the constant.         */
int tg_vec_compare_int(int device, int on_device, int op, int a_unsigned, int b_unsigned,
                       const tg_column* a, const tg_column* b, int64_t b_const,
                       int64_t* result, uint8_t* result_nulls, void* stream);
/* builtinLTRealSig etc (builtin_compare_vec_generated.go:54, cmp.Compare NaN ordering)        */
int tg_vec_compare_real(int device, int on_device, int op,
                        const tg_column* a, const tg_column* b, double b_const,
                        int64_t* result, uint8_t* result_nulls, void* stream);
/* builtinArithmeticPlusIntSig.vecEvalInt (builtin_arithmetic_vec.go:856-908, overflow :957),
 * MinusInt (:365, overflowCheck builtin_arithmetic.go:491), MultiplyInt / MultiplyIntUnsigned
 * (:646, :1011): the four signed/unsigned combinations; overflow on a non-NULL row ->
 * TG_ERR_OVERFLOW                                                                               */
int tg_vec_arith_int(int device, int on_device, int op, int a_unsigned, int b_unsigned,
                     const tg_column* a, const tg_column* b, int64_t b_const,
                     int64_t* result, uint8_t* result_nulls, void* stream);
/* builtinArithmeticPlusRealSig.vecEvalReal (:496-523), MinusReal, MultiplyReal:
 * +-Inf/NaN on a non-NULL row -> TG_ERR_OVERFLOW                                               */
int tg_vec_arith_real(int device, int on_device, int op,
                      const tg_column* a, const tg_column* b, double b_const,
                      double* result, uint8_t* result_nulls, void* stream);
/* expression.VectorizedFilter (chunk_executor.go:413) over a CNF of tg_filter_item:
 * selected[i] (1 byte per physical row, Go []bool) = all items true and not NULL.              */
int tg_vec_filter(int device, int on_device, const tg_chunk* chk,
                  const tg_filter_item* items, int32_t n_items,
                  uint8_t* selected, int64_t* n_selected, void* stream);

/* DECIMAL comparisons over 40-byte MyDecimal cells (the layout of tg_agg_func.ret_type), for Selection and Projection.
 *   Order: cells compare exactly as tg_topn orders DECIMAL cells, which is MyDecimal.Compare (types/mydecimal.go:1623):
 *     the sign first, so a cell with `negative` set and a zero value is below +0 and above every negative value; then the
 *     word magnitudes, integer words right-aligned and fraction words left-aligned on the point, leading and trailing
 *     zero words not counted, so 1.50 == 1.5 whatever the digitsInt.  resultFrac and the unused words are ignored.
 *   Any well-formed cell of any precision is accepted: no flen or scale is needed, so HAVING runs over SUM results wider
 *     than 18 digits.  A non-NULL cell is malformed when digitsInt or digitsFrac is negative, it has more than 9 integer
 *     and fraction words, or one of those words is >= 10^9 (tg_topn's definition).  Every non-NULL cell of a DECIMAL
 *     operand column is checked at every row the call evaluates (the rows in `sel` when the chunk has one, else every
 *     physical row), whatever the other items and the other operand give; one malformed cell fails the call with
 *     TG_ERR_INVALID.  Cells under NULL and outside `sel` are never read as values.  A malformed constant cell, a missing
 *     one, or an operand column whose elem_len is not 40 is TG_ERR_INVALID.
 *   Device-resident DECIMAL columns must be 8-byte aligned. */
/* tg_filter_item.is_real values understood by tg_vec_filter_ex */
enum { TG_FILTER_INT = 0, TG_FILTER_REAL = 1, TG_FILTER_DECIMAL = 2 };

/* builtin{LT,LE,GT,GE,EQ,NE}DecimalSig.vecEvalInt (expression/builtin_compare_vec_generated.go:64, :960, :1184):
 * result int64 0/1, NULL if either side is NULL (MergeNulls).  b == NULL -> compare with the 40-byte constant cell
 * b_const_cell (host memory).  A NULL row has its result bit cleared and the value 0. */
int tg_vec_compare_decimal(int device, int on_device, int op, const tg_column* a, const tg_column* b,
                           const uint8_t* b_const_cell, int64_t* result, uint8_t* result_nulls, void* stream);

/* tg_vec_filter plus DECIMAL items: col_types[c] is the MySQL type of chunk column c; an item with
 * is_real == TG_FILTER_DECIMAL compares 40-byte MyDecimal cells, against column rhs_col or, when rhs_col < 0, against
 * the constant cell at dec_consts + 40 * i (host memory; may be NULL when no DECIMAL item has a constant).
 *   A DECIMAL item needs col_types TG_TYPE_NEWDECIMAL and elem_len 40 on both operands.  A DECIMAL column in an INT or
 *   REAL item, or a column of another type in a DECIMAL item, is TG_ERR_UNSUPPORTED: the planner casts before it
 *   compares a DECIMAL with an integer or real operand.  INT and REAL items (is_real 0 / 1) keep exactly their
 *   tg_vec_filter meaning, so items of all kinds mix in one CNF of at most TG_MAX_FILTER (8) items over at most 16
 *   columns.  Any other is_real value, an op outside TG_CMP_*, or operand columns of different lengths is
 *   TG_ERR_INVALID.  With no DECIMAL item the call is tg_vec_filter: the same `selected` and count. */
int tg_vec_filter_ex(int device, int on_device, const tg_chunk* chk, const int32_t* col_types,
                     const tg_filter_item* items, int32_t n_items, const uint8_t* dec_consts,
                     uint8_t* selected, int64_t* n_selected, void* stream);

/* The form the two calls above compare a constant cell in (host code, no device): `out` gets the cell's sign and value
 * without leading zero integer words and trailing zero fraction words, digitsInt / digitsFrac = 9 * the words kept,
 * resultFrac and the unused words 0.  It compares with every cell as `cell` does.  A malformed cell is TG_ERR_INVALID
 * with `out` not written. */
int tg_decimal_normalize(const uint8_t* cell, uint8_t* out);

/* String comparisons and LIKE over var-length columns, for Selection and Projection.
 *   Columns: a string column is a chunk column with elem_len = -1, `offsets` of length + 1 int64 values and `data`
 *     (Column.GetString, pkg/util/chunk/column.go:715; the layout tg_chunk_decode returns).  Row r holds the bytes
 *     data[offsets[r] .. offsets[r+1]).  Offsets need not start at 0: a view into a larger buffer is valid, and the call
 *     reads only [offsets[0], offsets[length]).  In tg_vec_filter_ex2 its col_types entry is TG_TYPE_VARCHAR,
 *     TG_TYPE_VARSTRING, TG_TYPE_STRING or one of the four BLOB / TEXT types; ENUM, SET, JSON and BIT are var-length but
 *     not strings, so an item over them is TG_ERR_UNSUPPORTED.  Device-resident `data` and `offsets` need only their
 *     natural (1- and 8-byte) alignment.
 *   Offsets: checked at every row the call evaluates, NULL or not (the rows in `sel` when the chunk has one, else every
 *     physical row).  A row is bad when offsets[r] > offsets[r+1] or either value lies outside
 *     [offsets[0], offsets[length]]; a bad row fails the call with TG_ERR_INVALID.  With host columns,
 *     offsets[length] < offsets[0] is TG_ERR_INVALID.
 *   Collation: the MySQL collation id of the comparison (the builtin's collation), one of three collator behaviours
 *     (pkg/util/collate/bin.go, collate.go newCollatorIDMap):
 *       63 binary                                          compare: strings.Compare on the bytes; LIKE: over bytes
 *                                                          (CompilePatternBinary / DoMatchBinary)
 *       46 utf8mb4_bin, 83 utf8_bin, 65 ascii_bin, 47 latin1_bin
 *                                                          compare: strings.Compare after the trailing 0x20 bytes are cut
 *                                                          from both sides (truncateTailingSpace; a tab is kept, so
 *                                                          "a\t" > "a"); LIKE: over runes (CompilePattern / DoMatch),
 *                                                          trailing spaces count
 *       309 utf8mb4_0900_bin                               compare: strings.Compare on the bytes; LIKE: over runes
 *     Any other id (the _ci collations, gbk, gb18030) is TG_ERR_UNSUPPORTED.  Bytes compare unsigned; a proper prefix sorts
 *     first.
 *   LIKE: `column LIKE 'pattern' ESCAPE e` as builtinLikeSig.vecEvalInt (expression/builtin_like_vec.go) with a constant
 *     pattern and escape byte e (0..255, else TG_ERR_INVALID).  The escape is tested before '_' and '%' (so either may be
 *     the escape), an escape as the last character is a literal, "%%" is "%" and "%_" is "_%"; the match is
 *     stringutil.doMatchInner with its single restart point.  Over runes, the string and the pattern decode as Go's
 *     []rune(s): every byte that does not start a valid UTF-8 sequence (truncated, overlong, surrogate, above U+10FFFF)
 *     is one U+FFFD, so such bytes and a valid U+FFFD match each other, and the escape is the rune e (0xE9 is 'é', not
 *     the byte 0xE9).  A pattern from a column or a non-constant escape is not offloaded (the shim keeps the CPU path).
 *   The constant and the pattern have no length cap. */
enum { TG_FILTER_STRING = 3 };   /* tg_filter_item.is_real value understood by tg_vec_filter_ex2 */
enum { TG_STR_CMP = 0, TG_STR_LIKE = 1, TG_STR_NOT_LIKE = 2 };
typedef struct tg_str_arg {
  const uint8_t* bytes; int64_t len;  /* the constant (TG_STR_CMP with rhs_col < 0) or the LIKE pattern; host memory;
                                         may be NULL when len == 0                                                      */
  int32_t collation;                  /* MySQL collation id                                                             */
  int32_t kind;                       /* TG_STR_*; LIKE items ignore op and rhs_col                                     */
  int32_t escape;                     /* LIKE escape byte                                                               */
  int32_t reserved;
} tg_str_arg;

/* tg_vec_filter_ex plus STRING items (is_real == TG_FILTER_STRING): str_args[i] describes item i (read for STRING items
 * only; may be NULL when there is none).  A TG_STR_CMP item compares lhs_col with rhs_col or, when rhs_col < 0, with
 * the constant; TG_STR_LIKE / TG_STR_NOT_LIKE match lhs_col against the pattern.  NULL stays NULL, so a NOT LIKE item
 * does not select a NULL row.  STRING items mix with INT, REAL and DECIMAL items in one CNF of at most TG_MAX_FILTER (8)
 * items over at most 16 columns; a string column in a non-STRING item, or a non-string column in a STRING item, is
 * TG_ERR_UNSUPPORTED.  With no STRING item the call is tg_vec_filter_ex: the same `selected` and count. */
int tg_vec_filter_ex2(int device, int on_device, const tg_chunk* chk, const int32_t* col_types,
                      const tg_filter_item* items, int32_t n_items, const uint8_t* dec_consts,
                      const tg_str_arg* str_args, uint8_t* selected, int64_t* n_selected, void* stream);
/* builtin{LT,LE,GT,GE,EQ,NE}StringSig.vecEvalInt (expression/builtin_compare_vec_generated.go, types.CompareString):
 * result int64 0/1, NULL if either side is NULL (a NULL row's value is 0).  b == NULL -> compare with the constant
 * b_const[0 .. b_len) (host memory). */
int tg_vec_compare_string(int device, int on_device, int op, int32_t collation, const tg_column* a,
                          const tg_column* b, const uint8_t* b_const, int64_t b_len,
                          int64_t* result, uint8_t* result_nulls, void* stream);
/* builtinLikeSig.vecEvalInt with a constant pattern (host memory) and escape: result int64 0/1, NULL where a is NULL. */
int tg_vec_like(int device, int on_device, int32_t collation, const tg_column* a, const uint8_t* pattern,
                int64_t pattern_len, int32_t escape, int64_t* result, uint8_t* result_nulls, void* stream);

/* ---------------------------------------------------------------------------------------------
 * TopN                         replaces sortexec.TopNExec (pkg/executor/sortexec/topn.go:74, :230)
 * ORDER BY items over plain columns, LIMIT offset, count.  Rows [offset, offset + count) of the child's rows in item
 * order (NULL sorts before every value, DESC reverses: chunk.GetCompareFunc) are written to `out` (child schema, host
 * buffers, capacity >= min(count, rows - offset)); ties are broken arbitrarily, as by the reference's heap.
 * `on_device` as in the VecEval calls.  8-byte int-family / double / time columns, and DECIMAL columns of 40-byte
 * MyDecimal cells (elem_len 40 and col_types TG_TYPE_NEWDECIMAL; a 40-byte column of any other type, or an 8-byte column
 * typed NEWDECIMAL as an ORDER BY item, is TG_ERR_UNSUPPORTED), as ORDER BY items, payload or both.  These argument checks
 * need no device.  DOUBLE compares as Go cmp.Compare (NaN first, -0 == +0); DATE / DATETIME / TIMESTAMP compare by
 * calendar value and microseconds, ignoring the fsp and type bits (types/core_time.go compareTime).
 * DECIMAL compares as cmpMyDecimal / MyDecimal.Compare (types/mydecimal.go): the sign first, so a cell with `negative`
 * set and a zero value sorts after every negative value and before +0 (all such negative zeros are equal); then the
 * magnitudes by their words as doSub does: ceil(digitsInt / 9) integer words, then ceil(digitsFrac / 9) fraction words,
 * left-aligned, with leading zero integer words and trailing zero fraction words not counted (1.50 == 1.5 whatever the
 * digitsInt).  resultFrac and the words after the used ones are ignored.  Any well-formed cell of up to 9 words is
 * accepted, whatever its declared precision.  A non-NULL cell of a DECIMAL ORDER BY column is malformed when digitsInt
 * or digitsFrac is negative, its integer and fraction words number more than 9, or one of them is >= 10^9: every
 * non-NULL cell of such a column is checked (whatever offset and count select), and one malformed cell fails the call
 * with TG_ERR_INVALID, *nrows = 0 and `out` not written.  Payload cells are never interpreted.
 * The output rows keep the input's bits: a DECIMAL cell is copied whole (header, resultFrac and unused words included),
 * and a NULL row's cell is 40 zero bytes.  The output column of a DECIMAL column must have elem_len 40 (TG_ERR_INVALID
 * otherwise); device-resident DECIMAL columns must be 8-byte aligned.
 * ------------------------------------------------------------------------------------------- */
typedef struct tg_sort_item { int32_t col; int32_t desc; } tg_sort_item;
int tg_topn(int device, int on_device, const tg_chunk* chk, const int32_t* col_types, const uint32_t* col_flags,
            const tg_sort_item* items, int32_t n_items, int64_t offset, int64_t count,
            tg_mut_chunk* out, int64_t* nrows, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Key-hash repartition for the multi-GPU exchange (the GPU analogue of the MPP
 * ExchangeSender HashPartition, pkg/planner/core/operator/physicalop/physical_exchange_sender.go:115;
 * in-process analogue: partitionHashSplitter.split, pkg/executor/shuffle.go:450).
 * Device-resident: scatter `ncols` 8-byte columns of `rows` rows into `nparts` contiguous
 * regions by hash(key) (bits disjoint from the local table slot bits).  part_offsets receives
 * nparts+1 row offsets (device int64).  dst columns have capacity `rows`.  key_nulls_dev (bit 1 =
 * NOT NULL, LSB first; NULL = no NULL keys) only routes rows: a NULL key at row i goes to the
 * partition of hash(i).  No null bitmap is moved.
 * ------------------------------------------------------------------------------------------- */
int tg_partition_by_key(int device, const int64_t* key_dev, const uint8_t* key_nulls_dev,
                        int64_t rows, int32_t nparts, int32_t ncols,
                        const void* const* src_cols_dev, void* const* dst_cols_dev,
                        int64_t* part_offsets_dev, void* stream);
/* Same partition function evaluated on the host for one key (tests / planner)                 */
int32_t tg_partition_of_key(int64_t key, int32_t nparts);

/* Fused partition + NVLink exchange: like tg_partition_by_key but region p is written straight
 * into peer p's receive buffer (peer pointers mapped with tg_ipc_open) — the repartition step and
 * its all-to-all in one kernel.  recv_cols_peer[p*ncols + c] = device address (on peer p, mapped
 * here) of column c's receive buffer; recv_base[p] = first row this rank may write on peer p.   */
int tg_partition_exchange(int device, const int64_t* key_dev, int64_t rows, int32_t nparts,
                          int32_t ncols, const void* const* src_cols_dev,
                          void* const* recv_cols_peer, const int64_t* part_counts_dev,
                          const int64_t* recv_base_dev, void* stream);
/* Count-free variant (no histogram pass, no host round trip): every destination p owns, inside each receiver's
 * buffers, the fixed-capacity region [region_base, region_base + region_cap) reserved for THIS sender; rows are
 * appended there in arrival order and sent_rows_dev[p] (device, zeroed by the call) ends up holding how many rows went
 * to p.  sent_rows_dev[p] counts the rows destined to p, which can exceed region_cap; it is not the number of rows stored
 * there (receivers clamp it to region_cap).  A destination that would overflow raises *overflow_dev (device u64, sticky: the caller zeroes it once) and drops the excess —
 * the caller re-runs that step through tg_partition_count + tg_partition_exchange.  Returns after ENQUEUEING on `stream`.
 * The MPP analogue is still ExchangeSender/HashPartition (physical_exchange_sender.go:115); the reference sizes
 * its per-partition chunks dynamically on the host (shuffle.go:450), which a single GPU kernel cannot.            */
int tg_partition_exchange_cf(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                             const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                             int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev, void* stream);

/* tg_partition_exchange_cf with a cap on the scatter kernel's CTAs per SM (0 = as many as fit).  When the exchange
 * is NVLink-bound a few CTAs per SM already saturate the links, and the probe kernel of the previous step — running
 * next to it on another stream — keeps the SMs' L1 (the bulk-store scatter holds 49 KB of shared memory per CTA).   */
int tg_partition_exchange_cf_ex(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                                const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                                int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev, int32_t ctas_per_sm,
                                void* stream);

/* tg_partition_exchange_cf_ex whose destinations cannot lose rows to skew: a row that does not fit its destination's region
 * is appended to a LOCAL spill area instead (column c at spill_cols_dev[c], at most spill_cap rows in total, filled through
 * *spill_cursor_dev — device u64, zeroed by the caller, it keeps counting across calls).  After the pipeline the caller reads
 * the cursor once and moves the spilled rows with the counted exchange (tg_partition_count + tg_partition_exchange).
 * *overflow_dev is raised only when the spill area itself is full.  The reference's exchange has unbounded per-partition
 * queues (executor/shuffle.go:450) — skew makes it slower, never wrong; this is the fixed-capacity equivalent.           */
int tg_partition_exchange_cf_spill(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                                   const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                                   int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev,
                                   void* const* spill_cols_dev, int64_t spill_cap, uint64_t* spill_cursor_dev,
                                   int32_t ctas_per_sm, void* stream);

/* Transfer stage of the count-free exchange on the SMs instead of the copy engines: region r = the first
 * min(counts_dev[count_index[r]], cap_rows) rows (8 bytes each) of src_dev[r] -> dst_peer[r] (a peer address mapped with
 * tg_ipc_open).  128-bit loads / stores, no shared memory, <= 32 registers: the kernel fits NEXT TO the persistent probe
 * kernel on every SM and copies only the filled part of each region (the copy engines move whole regions: the host
 * never learns the fill).  ctas = 0: one 128-thread CTA per SM.                                                        */
#define TG_COPY_MAX_REGIONS 64
int tg_peer_copy_regions(int device, int32_t n_regions, const void* const* src_dev, void* const* dst_peer,
                         const int32_t* count_index, const int64_t* counts_dev, int64_t cap_rows, int32_t ctas, void* stream);

/* Cross-GPU mailboxes — the synchronisation of the count-free exchange without NCCL and without the host: one 8-byte
 * word per (sender) in a device buffer of the RECEIVER that every sender has mapped with tg_ipc_open.
 *   tg_mail_signal: after everything already enqueued on `stream` (the scatter kernel whose peer stores it publishes),
 *                   store  epoch << 40 | values_dev[p]  into targets->slot[p] for every p (values_dev NULL: 0).
 *   tg_mail_wait  : block `stream` (a spinning 32-thread kernel, the host never waits) until every one of the n words at
 *                   mail_dev carries an epoch >= `epoch`; the low 40 bits go to values_out_dev[p] (e.g. the fill count of
 *                   sender p's region = tg_join_probe_dev_seg's seg_cnt_dev).  A sender that stays silent for
 *                   `timeout_ms` (0 = 10 s) raises *error_flag_dev = 1 + p and the wait ends: the GPU is never hung.
 * The MPP analogue: the ExchangeReceiver waiting for every sender's stream end (the reference does it over gRPC).   */
#define TG_MAIL_MAX_PEERS 16
typedef struct tg_mail_targets { int32_t n, pad; uint64_t* slot[TG_MAIL_MAX_PEERS]; } tg_mail_targets;
int tg_mail_signal(int device, const tg_mail_targets* targets, const int64_t* values_dev, int64_t epoch, void* stream);
int tg_mail_wait(int device, const uint64_t* mail_dev, int32_t n, int64_t epoch, int64_t* values_out_dev,
                 uint64_t* error_flag_dev, int64_t timeout_ms, void* stream);

/* count rows per destination (first half of the exchange: counts are all-gathered by the host) */
int tg_partition_count(int device, const int64_t* key_dev, int64_t rows, int32_t nparts,
                       int64_t* part_counts_dev, void* stream);
/* cudaIpc handle plumbing for one-process-per-GPU peer access (64-byte opaque handle)           */
int tg_ipc_export(int device, void* dev_ptr, uint8_t handle_out[64]);
int tg_ipc_open(int device, const uint8_t handle[64], void** out_ptr);
int tg_ipc_close(int device, void* mapped_ptr);

#ifdef __cplusplus
}
#endif
#endif /* TIDBGPU_H */
