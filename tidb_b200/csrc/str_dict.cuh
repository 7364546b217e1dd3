// str_dict.cuh — device string dictionaries of the hash aggregation (str_dict.cu): a string GROUP BY column becomes a
// dense int64 id column before any update kernel sees it, so the group table, the DISTINCT sets and the finalize kernels
// treat it as an integer key.
//
// One dictionary per string GROUP BY column, in device memory for the life of the handle:
//   table   open-addressing records of 16 bytes {tag, id}; the tag is hash|3 when published, (hash & ~3)|1 while its
//           inserter writes the entry, 0 when empty (the multi-key group table's protocol)
//   entries by id: key bytes pointer, key length (the collation key: trailing 0x20 cut under a PAD collation), raw length
//           and the ordinal of the earliest row seen with the key
//   arena   the raw bytes of each entry's earliest row
// Entries live by id, so a growth rehashes 16-byte records from their stored tags (no bytes are read) and the result
// gather indexes the entries with the ids finalize wrote.
#pragma once
#include "common.cuh"

namespace tg {

// a tail value (k_str_dict_encode `tails`): (row ordinal << kTailBits) | trailing 0x20 bytes the PAD key cut
constexpr int kTailBits = 23;

// one var-length column of a batch on the device: row p holds the bytes data - base + [offs[p], offs[p + 1])
struct StrColDev { const int64_t* offs; const uint8_t* data; int64_t base; const uint8_t* nulls; };

struct StrDict {
  int coll = 0;                       // StrColl (string.cuh) of the column's collation
  DevBuf tbl;                         // nslots records {tag, id}
  unsigned long long nslots = 0;
  DevBuf kptr, klen, rlen, first;     // per id
  size_t id_cap = 0;
  DevBuf arena;
  size_t arena_used = 0;
  DevBuf ctr;                         // [0] entries, [1] rows deferred, [2] bytes of the new entries, [3] arena cursor,
                                      // [4] entries taken or being taken, [5] rows deferred by a long probe, [6] a
                                      // trailing-space count too wide for kTailBits
  int64_t entries = 0, grows = 0, launches = 0;
};

// bad-offsets check of n device rows (every row, NULL or not): *flag = 1 when a row has offs[r] > offs[r + 1], a value
// outside [offs[0], offs[n]], or bytes while data is NULL.  Enqueued on s; the caller reads the flag back.
void str_check_offsets(const int64_t* offs, const uint8_t* data, int64_t n, unsigned int* flag, int nsm, cudaStream_t s);

// before the rounds of a batch of n rows: the table exists (first one: twice min(n, 4 M) slots, at least 1024, bounded
// by twice expected_groups when given) and the entry arrays have room for 1024 more entries (half the table's slots at
// first); a round defers new entries that find no room, and str_dict_grow makes it
int str_dict_prepare(StrDict& d, int device, int64_t n, int64_t expected_groups, cudaStream_t s);

// one encode round over the batch (only == nullptr: every row, else the rows whose bit is set): ids[i] = the id of row
// i's key, 0 for a NULL row; a row whose probe runs past max_probe is deferred (its bit set in `deferred`), nd = their
// number.  ord0 + i is row i's ordinal (push order).  tails (may be nullptr): per row (ordinal << kTailBits) | the
// trailing spaces the PAD key cut; a count of 2^kTailBits or more sets ctr[6] (str_dict_tail_overflow).
int str_dict_round(StrDict& d, const StrColDev& c, int64_t n, int64_t ord0, uint32_t max_probe, long long* ids, uint32_t* deferred,
                   const uint32_t* only, unsigned long long& nd, unsigned long long* tails, int nsm, cudaStream_t s);

// true when the last batch's tails had a trailing-space count that does not fit kTailBits
int str_dict_tail_overflow(StrDict& d, bool& overflow, cudaStream_t s);

// the entries the table holds, this batch's new ones included
int str_dict_used(StrDict& d, unsigned long long& used, cudaStream_t s);

// after a round deferred rows: x4 room in the per-id arrays when new entries found none, and, unless the table has room
// (the next round walks it without a probe limit), a rehash into a table x4 bigger, or half full with `more` new
// entries, when a probe ran past its limit
int str_dict_grow(StrDict& d, unsigned long long more, bool room, int device, int nsm, cudaStream_t s);

// after the last round: each new entry takes the raw bytes of its earliest row of the batch into the arena, so that no
// entry points into the batch's buffers any more
int str_dict_commit(StrDict& d, const StrColDev& c, const long long* ids, int64_t n, int64_t ord0, int device, int nsm, cudaStream_t s);

// result column of `rows` ids (valid[r] == 0: NULL, a 0-length row; valid may be nullptr): offs (rows + 1, from 0) and
// bytes; *total = offs[rows].  Row r is its entry's raw bytes, or with tails (the groups' MIN of the tail values) the
// entry's key bytes followed by tails[r]'s count of spaces: the raw bytes of the group's own earliest row.
int str_dict_gather(const StrDict& d, const long long* ids, const uint8_t* valid, const unsigned long long* tails, int64_t rows, DevBuf& offs, DevBuf& bytes,
                    int64_t* total, int device, int nsm, cudaStream_t s);

}  // namespace tg
