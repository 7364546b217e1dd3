// oracle/join.cpp — CPU restatement of HashJoinV2Exec (TEST INFRASTRUCTURE, see oracle.h).
//
// Follows, function by function, the reference's Go sources under pkg/executor/join:
//   join_table_meta.go   newTableMeta :184, setupJoinKeys :260, setupColumnOrder :331, getKeyProp :130
//   row_table_builder.go processOneChunk :138, initHashValueAndPartIndexForOneChunk :103,
//                        appendToRowTable :530, fillNullMap :375, fillRowData :433
//   join_row_table.go    row layout :81-105, getNextRowAddress :162
//   hash_table_v2.go     newSubTable :67, updateHashValue :85, atomicUpdateHashValue :94, lookup :45
//   tagged_ptr.go        tagPtrHelper :40-70
//   hash_join_v2.go      genHashJoinPartitionNumber :298, getPartitionMaskOffset :306, worker
//                        structure :1266-1479 (build) and :793-852 (probe)
//   base_join_probe.go   SetChunkForProbe :179, isKeyMatched :820, NewJoinProbe :850
//   inner_join_probe.go :27, outer_join_probe.go :250/:308/:117, semi_join_probe.go,
//   anti_semi_join_probe.go, left_outer_semi_join_probe.go
// and pkg/util/codec/codec.go SerializeKeys :822 / serializeKeysImpl :622.
//
// Scope: fixed-width columns (elem_len 4/8/40), integer-family / float / double join keys (one or
// many), build/probe filters as tg_filter_item CNF, OtherCondition as tg_other_item CNF on candidate pairs
// (inner_join_probe.go:72-79 / base_join_probe.go:758, for the join shapes the GPU gate accepts), no spill.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <memory>
#include <thread>
#include <map>
#include <set>
#include "common.hpp"

namespace orc {

// ------------------------------------------------------------------------------------------------
// primitives
// ------------------------------------------------------------------------------------------------
static const uint64_t kFnvOffset64 = 14695981039346656037ull;  // Go hash/fnv offset64
static const uint64_t kFnvPrime64 = 1099511628211ull;          // Go hash/fnv prime64

// Go hash/fnv (*sum64).Write: hash *= prime64; hash ^= byte   (FNV-1)
inline uint64_t fnv1_64(const uint8_t* p, size_t n) {
  uint64_t h = kFnvOffset64;
  for (size_t i = 0; i < n; i++) { h *= kFnvPrime64; h ^= (uint64_t)p[i]; }
  return h;
}

// hash_table_v2.go:55
inline uint64_t next_power_of_two(uint64_t value) {
  uint64_t ret = 2;
  int round = 1;
  for (; ret <= value && round <= 64; ret <<= 1) round++;
  return ret;
}
// hash_join_v2.go:298
inline uint32_t gen_partition_number(uint32_t hint) {
  uint32_t p = 1;
  while (p < hint && p < 16) p <<= 1;
  return p;
}
// hash_join_v2.go:306 — 64 - trailingZeros(partitionNumber)
inline int partition_mask_offset(uint32_t pn) { return 64 - __builtin_ctzll((uint64_t)pn); }
// Go shifts >= width yield 0 (hash_join_v2.go:1487 generatePartitionIndex)
inline uint64_t partition_index(uint64_t h, int off) { return off >= 64 ? 0 : (h >> off); }

// tagged_ptr.go
static const int8_t kMaxTaggedBits = 24;
inline uint8_t tagged_bits_from_ptr(uint64_t p) {
  int lz = p == 0 ? 64 : __builtin_clzll(p);
  return (uint8_t)std::min<int>(lz, kMaxTaggedBits);
}
struct TagHelper {
  uint64_t mask = 0;
  void init(uint8_t bits) {
    uint64_t m = bits >= 64 ? ~0ull : ((1ull << bits) - 1);
    int off = 64 - bits;
    mask = bits == 0 ? 0 : (m << off);
  }
  uint64_t tag_of(uint64_t h) const { return h & mask; }
  uint64_t to_tagged(uint64_t tag, const uint8_t* p) const { return (uint64_t)(uintptr_t)p | tag; }
  uint8_t* to_ptr(uint64_t t) const { return (uint8_t*)(uintptr_t)(t & ~mask); }
};

// ------------------------------------------------------------------------------------------------
// joinTableMeta (join_table_meta.go)
// ------------------------------------------------------------------------------------------------
enum KeyMode { OneInt64 = 0, FixedSerializedKey = 1, VariableSerializedKey = 2 };
enum SerializeMode { Normal = 0, NeedSignFlag = 1, KeepVarColumnLength = 2 };
static const int sizeOfNextPtr = 8;
static const int sizeOfElementSize = 4;

struct KeyProp { bool canBeInlined; int keyLength; bool isKeyInteger; bool isKeyUnsigned; };

// join_table_meta.go:130 getKeyProp
static KeyProp get_key_prop(const FieldType& tp) {
  switch (tp.tp) {
    case TypeTiny: case TypeShort: case TypeInt24: case TypeLong: case TypeLonglong: case TypeYear:
    case TypeDuration: {
      bool uns = (tp.flag & UnsignedFlag) != 0;
      if (tp.tp == TypeYear) uns = true;
      else if (tp.tp == TypeDuration) uns = false;
      return {true, fixed_len(tp.tp), true, uns};
    }
    case TypeVarchar: case TypeVarString: case TypeString: case TypeBlob: case TypeTinyBlob:
    case TypeMediumBlob: case TypeLongBlob:
      return {tp.binary_coll, VarElemLen, false, false};
    case TypeDate: case TypeDatetime: case TypeTimestamp:
      return {false, 8, true, true};
    case TypeFloat:
      return {false, 8, false, false};
    case TypeNewDecimal:
      return {false, VarElemLen, false, false};
    case TypeEnum:
      if (tp.flag & EnumSetAsIntFlag) return {false, 8, true, true};
      return {false, VarElemLen, false, false};
    case TypeBit:
      return {false, 8, true, true};
    default:
      return {false, fixed_len(tp.tp), false, false};
  }
}

struct Meta {
  bool isFixedLength = true;
  int rowLength = 0;
  bool isJoinKeysFixedLength = true;
  int joinKeysLength = 0;
  bool isJoinKeysInlined = true;
  int nullMapLength = 0;
  std::vector<int> rowColumnsOrder;
  std::vector<int> columnsSize;
  std::vector<int> serializeModes;
  int columnCountNeededForOtherCondition = 0;
  int totalColumnNumber = 0;
  int colOffsetInNullMap = 0;
  int keyMode = OneInt64;
  int rowDataOffset = -1;
  std::vector<uint8_t> fakeKeyByte;
};

// join_table_meta.go:260 setupJoinKeys
static void setup_join_keys(Meta& meta, const std::vector<int>& buildKeyIndex,
                            const std::vector<FieldType>& buildKeyTypes,
                            const std::vector<FieldType>& probeKeyTypes) {
  meta.isJoinKeysFixedLength = true;
  meta.joinKeysLength = 0;
  meta.isJoinKeysInlined = true;
  meta.serializeModes.clear();
  bool isAllKeyInteger = true;
  int varLengthKeyNumber = 0;
  std::set<int> keyIndexMap;
  for (size_t index = 0; index < buildKeyIndex.size(); index++) {
    KeyProp prop = get_key_prop(buildKeyTypes[index]);
    if (prop.keyLength != VarElemLen) meta.joinKeysLength += prop.keyLength;
    else { meta.isJoinKeysFixedLength = false; varLengthKeyNumber++; }
    if (!prop.canBeInlined) meta.isJoinKeysInlined = false;
    if (prop.isKeyInteger) {
      KeyProp pp = get_key_prop(probeKeyTypes[index]);
      if (prop.isKeyUnsigned != pp.isKeyUnsigned) {
        meta.serializeModes.push_back(NeedSignFlag);
        meta.isJoinKeysInlined = false;
        if (meta.isJoinKeysFixedLength) meta.joinKeysLength++;
      } else {
        meta.serializeModes.push_back(Normal);
      }
    } else {
      isAllKeyInteger = false;
      if (prop.keyLength == VarElemLen) meta.serializeModes.push_back(KeepVarColumnLength);
      else meta.serializeModes.push_back(Normal);
    }
    keyIndexMap.insert(buildKeyIndex[index]);
  }
  if (!meta.isJoinKeysFixedLength) meta.joinKeysLength = -1;
  if (buildKeyIndex.size() != keyIndexMap.size()) meta.isJoinKeysInlined = false;
  if (!meta.isJoinKeysInlined && varLengthKeyNumber == 1) {
    for (auto& m : meta.serializeModes) if (m == KeepVarColumnLength) m = Normal;
  }
  if (isAllKeyInteger && buildKeyIndex.size() == 1 && meta.serializeModes[0] != NeedSignFlag) {
    meta.keyMode = OneInt64;
  } else {
    meta.keyMode = meta.isJoinKeysFixedLength ? FixedSerializedKey : VariableSerializedKey;
  }
}

// join_table_meta.go:184 newTableMeta.  other / output == nullptr restates Go nil.
static Meta new_table_meta(const std::vector<int>& buildKeyIndex, const std::vector<FieldType>& buildTypes,
                           const std::vector<FieldType>& buildKeyTypes,
                           const std::vector<FieldType>& probeKeyTypes,
                           const std::vector<int>* other, const std::vector<int>* output,
                           bool needUsedFlag) {
  Meta meta;
  meta.totalColumnNumber = (int)buildTypes.size();
  std::set<int> saved;
  auto updateMeta = [&](int index) {
    if (saved.insert(index).second) {
      int length = fixed_len(buildTypes[index].tp);
      if (length == VarElemLen) meta.isFixedLength = false;
      else meta.rowLength += length;
    }
  };
  if (!output) {
    for (size_t i = 0; i < buildTypes.size(); i++) updateMeta((int)i);
  } else {
    for (int i : *output) updateMeta(i);
    if (other) for (int i : *other) updateMeta(i);
  }
  setup_join_keys(meta, buildKeyIndex, buildKeyTypes, probeKeyTypes);
  if (meta.isJoinKeysInlined) for (int i : buildKeyIndex) updateMeta(i);
  if (!meta.isFixedLength) meta.rowLength = 0;
  int savedColumnNum = (int)saved.size();

  // setupColumnOrder :331
  std::set<int> used;
  auto updateOrder = [&](int index) {
    if (used.insert(index).second) {
      meta.rowColumnsOrder.push_back(index);
      meta.columnsSize.push_back(fixed_len(buildTypes[index].tp));
    }
  };
  if (meta.isJoinKeysInlined) for (int i : buildKeyIndex) updateOrder(i);
  meta.columnCountNeededForOtherCondition = 0;
  if (other && !other->empty()) {
    for (int i : *other) updateOrder(i);
    meta.columnCountNeededForOtherCondition = (int)used.size();
  }
  if (!output) { for (size_t i = 0; i < buildTypes.size(); i++) updateOrder((int)i); }
  else for (int i : *output) updateOrder(i);

  if (needUsedFlag) {
    meta.colOffsetInNullMap = 1;
    meta.nullMapLength = ((savedColumnNum + 1 + 31) / 32) * 4;
  } else {
    meta.colOffsetInNullMap = 0;
    meta.nullMapLength = (savedColumnNum + 7) / 8;
  }
  meta.rowDataOffset = -1;
  if (meta.isJoinKeysInlined) {
    meta.rowDataOffset = meta.isJoinKeysFixedLength ? sizeOfNextPtr + meta.nullMapLength
                                                    : sizeOfNextPtr + meta.nullMapLength + sizeOfElementSize;
  } else if (meta.isJoinKeysFixedLength) {
    meta.rowDataOffset = sizeOfNextPtr + meta.nullMapLength + meta.joinKeysLength;
  }
  if (meta.isJoinKeysFixedLength && !meta.isJoinKeysInlined) meta.fakeKeyByte.assign(meta.joinKeysLength, 0);
  return meta;
}

// usedFlagMask: join_table_meta.go — the first bit (MSB of byte 0) of the null map read as a
// little-endian uint32; the reference computes it at init from a byte pattern {0x80,0,0,0}.
static const uint32_t kUsedFlagMask = 0x80u;

// ------------------------------------------------------------------------------------------------
// row tables and hash tables
// ------------------------------------------------------------------------------------------------
struct Segment {   // rowTableSegment join_row_table.go:81
  std::vector<uint8_t> rawData;
  std::vector<uint64_t> hashValues;
  std::vector<uint64_t> rowStartOffset;
  std::vector<int> validJoinKeyPos;
  uint8_t taggedBits = 0;
  uint8_t* row_ptr(size_t i) { return rawData.data() + rowStartOffset[i]; }
  void init_tagged_bits() {   // join_row_table.go:129
    uint64_t s = (uint64_t)(uintptr_t)row_ptr(0);
    uint64_t e = (uint64_t)(uintptr_t)row_ptr(rowStartOffset.size() - 1);
    taggedBits = tagged_bits_from_ptr(s | e);
  }
};

struct SubTable {   // hash_table_v2.go:22
  std::vector<Segment*> segments;
  std::vector<std::atomic<uint64_t>> hashTable;
  uint64_t posMask = 0;
  uint64_t row_count() const { uint64_t n = 0; for (auto* s : segments) n += s->rowStartOffset.size(); return n; }
  uint64_t valid_key_count() const { uint64_t n = 0; for (auto* s : segments) n += s->validJoinKeyPos.size(); return n; }
  void alloc() {   // newSubTable :67
    uint64_t len = std::max<uint64_t>(next_power_of_two(valid_key_count()), 32);
    hashTable = std::vector<std::atomic<uint64_t>>(len);
    for (auto& x : hashTable) x.store(0, std::memory_order_relaxed);
    posMask = len - 1;
  }
  static void set_next(uint8_t* row, uint64_t next) { std::memcpy(row, &next, 8); }
  // updateHashValue :85
  void update(uint64_t h, uint8_t* row, const TagHelper& th) {
    uint64_t pos = h & posMask;
    uint64_t prev = hashTable[pos].load(std::memory_order_relaxed);
    uint64_t tag = th.tag_of(h | prev);
    hashTable[pos].store(th.to_tagged(tag, row), std::memory_order_relaxed);
    set_next(row, prev);
  }
  // atomicUpdateHashValue :94
  void atomic_update(uint64_t h, uint8_t* row, const TagHelper& th) {
    uint64_t pos = h & posMask;
    for (;;) {
      uint64_t prev = hashTable[pos].load();
      uint64_t tag = th.tag_of(h | prev);
      uint64_t tagged = th.to_tagged(tag, row);
      if (hashTable[pos].compare_exchange_strong(prev, tagged)) { set_next(row, prev); break; }
    }
  }
  // build :107
  void build(size_t segStart, size_t segEnd, const TagHelper& th) {
    bool single = (segStart == 0 && segEnd == segments.size());
    for (size_t i = segStart; i < segEnd; i++) {
      Segment* s = segments[i];
      for (int idx : s->validJoinKeyPos) {
        if (single) update(s->hashValues[idx], s->row_ptr(idx), th);
        else atomic_update(s->hashValues[idx], s->row_ptr(idx), th);
      }
    }
  }
  // lookup :45
  uint64_t lookup(uint64_t h, const TagHelper& th) const {
    uint64_t ret = hashTable[h & posMask].load(std::memory_order_relaxed);
    uint64_t tag = th.tag_of(h);
    if ((ret & tag) != tag) return 0;
    return ret;
  }
};

// getNextRowAddress join_row_table.go:162
inline uint64_t next_row_address(const uint8_t* row, const TagHelper& th, uint64_t h) {
  uint64_t ret; std::memcpy(&ret, row, 8);
  uint64_t tag = th.tag_of(h);
  if ((ret & tag) != tag) return 0;
  return ret;
}

// ------------------------------------------------------------------------------------------------
// codec.SerializeKeys (util/codec/codec.go:822 → serializeKeysImpl :622) for one chunk
// ------------------------------------------------------------------------------------------------
struct SerializedKeys {
  std::vector<uint8_t> buf;
  std::vector<uint32_t> off;    // per logical row start; len = off[i+1]-off[i]
  const uint8_t* key(size_t i) const { return buf.data() + off[i]; }
  size_t len(size_t i) const { return off[i + 1] - off[i]; }
};

static const uint8_t intFlag = 3, uintFlag = 4;   // codec.go:43-44

static bool serialize_keys(const tg_chunk& chk, const std::vector<FieldType>& tps,
                           const std::vector<int>& keyIdx, const std::vector<int64_t>& usedRows,
                           const std::vector<uint8_t>* filterVector, std::vector<uint8_t>* nullVector,
                           const std::vector<int>& modes, SerializedKeys& out) {
  size_t n = usedRows.size();
  // preAllocForSerializedKeyBuffer :429-447: NULL in any key column marks nullVector[physical]
  for (size_t k = 0; k < keyIdx.size(); k++) {
    const tg_column& col = chk.cols[keyIdx[k]];
    if (col.null_bitmap && nullVector) {
      for (size_t l = 0; l < n; l++) if (col_is_null(col, usedRows[l])) (*nullVector)[usedRows[l]] = 1;
    }
  }
  out.buf.clear(); out.off.assign(n + 1, 0);
  for (size_t l = 0; l < n; l++) {
    int64_t p = usedRows[l];
    out.off[l] = (uint32_t)out.buf.size();
    bool skip = (filterVector && !(*filterVector)[p]) || (nullVector && (*nullVector)[p]);
    if (skip) continue;
    for (size_t k = 0; k < keyIdx.size(); k++) {
      const tg_column& col = chk.cols[keyIdx[k]];
      const FieldType& tp = tps[k];
      switch (tp.tp) {
        case TypeTiny: case TypeShort: case TypeInt24: case TypeLong: case TypeLonglong: case TypeYear:
        case TypeDuration: {   // Duration: codec.go serializes GetRaw as well
          if (modes[k] == NeedSignFlag) {
            int64_t v = col_i64(col, p);
            if (!(tp.flag & UnsignedFlag) && v < 0) out.buf.push_back(intFlag);
            else out.buf.push_back(uintFlag);
          }
          const uint8_t* r = col_raw(col, p);
          out.buf.insert(out.buf.end(), r, r + 8);
          break;
        }
        case TypeFloat: {
          double d = (double)col_f32(col, p);
          if (d == 0) d = 0;   // -0 → +0, codec.go:663-667
          const uint8_t* r = reinterpret_cast<const uint8_t*>(&d);
          out.buf.insert(out.buf.end(), r, r + 8);
          break;
        }
        case TypeDouble: {
          double f = col_f64(col, p);
          if (f == 0) f = 0;   // codec.go:676-682
          const uint8_t* r = reinterpret_cast<const uint8_t*>(&f);
          out.buf.insert(out.buf.end(), r, r + 8);
          break;
        }
        case TypeDate: case TypeDatetime: case TypeTimestamp: {
          // codec.go:697-707: Time.ToPackedUint (types/time.go:646-657) of the CoreTime bit fields (types/time.go:235-241)
          const uint64_t v = (uint64_t)col_i64(col, p);
          const uint64_t year = (v >> 50) & 0x3fff, month = (v >> 46) & 0xf, day = (v >> 41) & 0x1f, hour = (v >> 36) & 0x1f,
                         minute = (v >> 30) & 0x3f, second = (v >> 24) & 0x3f, micro = (v >> 4) & 0xfffff;
          uint64_t packed = 0;
          if (year | month | day | hour | minute | second | micro) {   // IsZero → 0
            const uint64_t ymd = ((year * 13 + month) << 5) | day, hms = (hour << 12) | (minute << 6) | second;
            packed = (((ymd << 17) | hms) << 24) | micro;
          }
          const uint8_t* r = reinterpret_cast<const uint8_t*>(&packed);
          out.buf.insert(out.buf.end(), r, r + 8);
          break;
        }
        default:
          set_error("oracle: join key type not restated (var-len / decimal keys are out of scope)");
          return false;
      }
    }
  }
  out.off[n] = (uint32_t)out.buf.size();
  return true;
}

// ------------------------------------------------------------------------------------------------
// the join context
// ------------------------------------------------------------------------------------------------
struct Join {
  // descriptor
  int joinType = TG_JOIN_INNER;
  bool rightAsBuild = true;
  std::vector<FieldType> leftTypes, rightTypes;
  std::vector<int> leftKeyIdx, rightKeyIdx;
  std::vector<int> lUsed, rUsed;
  std::vector<tg_filter_item> buildFilter, probeFilter;
  std::vector<tg_other_item> otherCond;          // sides as given: 0 = left child, 1 = right child
  std::vector<int> otherBuildCols;               // build columns OtherCondition reads (stored first in the row, join_table_meta.go:217)
  uint32_t concurrency = 5;
  // derived
  std::vector<FieldType> buildTypes, probeTypes, buildKeyTypes, probeKeyTypes;
  std::vector<int> buildKeyIdx, probeKeyIdx;
  std::vector<int> buildUsed, probeUsed;   // output columns taken from the build / probe child
  int buildColOffsetInResult = 0, probeColOffsetInResult = 0;
  bool needScanRowTable = false;   // JoinProbe.NeedScanRowTable
  bool buildHasNullableKey = false, probeHasNullableKey = false;
  Meta meta;
  uint32_t partitionNumber = 1;
  int partitionMaskOffset = 64;
  TagHelper tagHelper;
  // row tables: [worker][partition] -> segments (hashTableContext.rowTables)
  std::vector<std::vector<std::vector<std::unique_ptr<Segment>>>> rowTables;
  std::vector<SubTable> tables;
  // results, one set of columns per probe worker
  int nOutCols = 0;
  std::vector<int> outElemLen;
  std::vector<std::vector<OColumn>> results;
  double buildSeconds = 0, probeSeconds = 0;
};

static bool is_left_side_build(const Join& j) { return !j.rightAsBuild; }

static bool setup_join(Join& j, std::string& err) {
  if (j.rightAsBuild) {
    j.buildTypes = j.rightTypes; j.probeTypes = j.leftTypes;
    j.buildKeyIdx = j.rightKeyIdx; j.probeKeyIdx = j.leftKeyIdx;
    j.buildUsed = j.rUsed; j.probeUsed = j.lUsed;
    j.buildColOffsetInResult = (int)j.lUsed.size(); j.probeColOffsetInResult = 0;
  } else {
    j.buildTypes = j.leftTypes; j.probeTypes = j.rightTypes;
    j.buildKeyIdx = j.leftKeyIdx; j.probeKeyIdx = j.rightKeyIdx;
    j.buildUsed = j.lUsed; j.probeUsed = j.rUsed;
    j.buildColOffsetInResult = 0; j.probeColOffsetInResult = (int)j.lUsed.size();
  }
  for (int k : j.buildKeyIdx) j.buildKeyTypes.push_back(j.buildTypes[k]);
  for (int k : j.probeKeyIdx) j.probeKeyTypes.push_back(j.probeTypes[k]);
  for (auto& t : j.buildKeyTypes) if (!(t.flag & NotNullFlag)) j.buildHasNullableKey = true;
  for (auto& t : j.probeKeyTypes) if (!(t.flag & NotNullFlag)) j.probeHasNullableKey = true;

  // NewJoinProbe base_join_probe.go:850-932: which probe type, and NeedScanRowTable
  switch (j.joinType) {
    case TG_JOIN_INNER: j.needScanRowTable = false; break;
    case TG_JOIN_LEFT_OUTER: j.needScanRowTable = !j.rightAsBuild; break;    // isOuterSideBuild
    case TG_JOIN_RIGHT_OUTER: j.needScanRowTable = j.rightAsBuild; break;
    case TG_JOIN_SEMI: case TG_JOIN_ANTI_SEMI:
      if (!j.rUsed.empty()) { err = "len(rUsed) != 0 for semi join"; return false; }
      j.needScanRowTable = is_left_side_build(j); break;
    case TG_JOIN_LEFT_OUTER_SEMI: case TG_JOIN_ANTI_LEFT_OUTER_SEMI:
      if (!j.rUsed.empty()) { err = "len(rUsed) != 0 for left outer semi join"; return false; }
      if (!j.rightAsBuild) { err = "unsupported join type (left outer semi needs right build)"; return false; }
      j.needScanRowTable = false; break;
    default: err = "unsupported join type"; return false;
  }
  // OpenSelf hash_join_v2.go:700-711
  if (!j.otherCond.empty()) {
    if (j.needScanRowTable || j.joinType == TG_JOIN_LEFT_OUTER_SEMI || j.joinType == TG_JOIN_ANTI_LEFT_OUTER_SEMI ||
        ((j.joinType == TG_JOIN_SEMI || j.joinType == TG_JOIN_ANTI_SEMI) && is_left_side_build(j))) {
      err = "oracle: OtherCondition is restated for inner / probe-side outer / right-build semi and anti-semi joins only"; return false;
    }
    for (const tg_other_item& it : j.otherCond) {
      for (int q = 0; q < 2; q++) {
        int side = q ? it.rhs_side : it.lhs_side, col = q ? it.rhs_col : it.lhs_col;
        if (side < 0) continue;
        bool is_build = (side == 1) == j.rightAsBuild;
        if (is_build && std::find(j.otherBuildCols.begin(), j.otherBuildCols.end(), col) == j.otherBuildCols.end()) j.otherBuildCols.push_back(col);
      }
    }
  }
  j.meta = new_table_meta(j.buildKeyIdx, j.buildTypes, j.buildKeyTypes, j.probeKeyTypes,
                          j.otherCond.empty() ? nullptr : &j.otherBuildCols, &j.buildUsed, j.needScanRowTable);
  if (!j.meta.isFixedLength || !j.meta.isJoinKeysFixedLength) {
    err = "oracle: var-len columns/keys are out of scope"; return false;
  }
  j.partitionNumber = gen_partition_number(j.concurrency);
  j.partitionMaskOffset = partition_mask_offset(j.partitionNumber);
  // output schema
  j.nOutCols = (int)(j.lUsed.size() + j.rUsed.size());
  j.outElemLen.clear();
  for (int c : j.lUsed) j.outElemLen.push_back(fixed_len(j.leftTypes[c].tp));
  for (int c : j.rUsed) j.outElemLen.push_back(fixed_len(j.rightTypes[c].tp));
  if (j.joinType == TG_JOIN_LEFT_OUTER_SEMI || j.joinType == TG_JOIN_ANTI_LEFT_OUTER_SEMI) {
    j.nOutCols += 1; j.outElemLen.push_back(8);   // the matched-flag column (int64, nullable)
  }
  return true;
}

// ------------------------------------------------------------------------------------------------
// build side: rowTableBuilder.processOneChunk
// ------------------------------------------------------------------------------------------------
static void used_rows_of(const tg_chunk& chk, std::vector<int64_t>& used) {
  int64_t n = chunk_logical_rows(chk);
  used.resize(n);
  if (chk.sel) for (int64_t i = 0; i < n; i++) used[i] = chk.sel[i];
  else for (int64_t i = 0; i < n; i++) used[i] = i;
}

static bool build_process_one_chunk(Join& j, const tg_chunk& chk, int workerID) {
  std::vector<int64_t> usedRows; used_rows_of(chk, usedRows);
  if (usedRows.empty()) return true;
  int64_t physicalRows = chunk_physical_rows(chk);
  bool hasFilter = !j.buildFilter.empty();
  std::vector<uint8_t> filterVector, nullKeyVector;
  if (hasFilter) {
    filterVector.resize(physicalRows);
    for (int64_t p = 0; p < physicalRows; p++)
      filterVector[p] = filter_row(chk, p, j.buildFilter.data(), (int)j.buildFilter.size());
  }
  if (j.buildHasNullableKey) nullKeyVector.assign(physicalRows, 0);
  SerializedKeys keys;
  if (!serialize_keys(chk, j.buildKeyTypes, j.buildKeyIdx, usedRows, hasFilter ? &filterVector : nullptr,
                      j.buildHasNullableKey ? &nullKeyVector : nullptr, j.meta.serializeModes, keys))
    return false;
  // initHashValueAndPartIndexForOneChunk :103
  size_t n = usedRows.size();
  std::vector<uint64_t> hashValue(n);
  std::vector<int> partIdx(n);
  uint64_t fakePartIndex = 0;
  for (size_t l = 0; l < n; l++) {
    int64_t p = usedRows[l];
    if ((hasFilter && !filterVector[p]) || (j.buildHasNullableKey && nullKeyVector[p])) {
      hashValue[l] = fakePartIndex; partIdx[l] = (int)fakePartIndex;
      fakePartIndex = (fakePartIndex + 1) % j.partitionNumber;
      continue;
    }
    uint64_t h = fnv1_64(keys.key(l), keys.len(l));
    hashValue[l] = h;
    partIdx[l] = (int)partition_index(h, j.partitionMaskOffset);
  }
  // appendToRowTable :530 (with preAllocForSegments :483 sizing so that row pointers stay stable)
  const Meta& meta = j.meta;
  bool keepFilteredRows = j.needScanRowTable;
  std::vector<std::unique_ptr<Segment>> segs(j.partitionNumber);
  std::vector<int64_t> rawLen(j.partitionNumber, 0), rowNum(j.partitionNumber, 0);
  auto row_length_of = [&](bool hasValidKey, size_t l) {
    int64_t len = sizeOfNextPtr + meta.nullMapLength;
    if (!meta.isJoinKeysFixedLength) len += sizeOfElementSize;
    if (!meta.isJoinKeysInlined) {
      if (hasValidKey) len += (int64_t)keys.len(l);
      else if (meta.isJoinKeysFixedLength) len += meta.joinKeysLength;
    }
    for (int sz : meta.columnsSize) len += sz;
    len += (8 - len % 8) % 8;   // calculateFakeLength :473
    return len;
  };
  for (size_t l = 0; l < n; l++) {
    int64_t p = usedRows[l];
    bool hasValidKey = (!hasFilter || filterVector[p]) && (!j.buildHasNullableKey || !nullKeyVector[p]);
    if (!hasValidKey && !keepFilteredRows) continue;
    rowNum[partIdx[l]]++;
    rawLen[partIdx[l]] += row_length_of(hasValidKey, l);
  }
  for (uint32_t pi = 0; pi < j.partitionNumber; pi++) {
    segs[pi].reset(new Segment());
    segs[pi]->rawData.reserve((size_t)rawLen[pi]);
    segs[pi]->hashValues.reserve((size_t)rowNum[pi]);
    segs[pi]->rowStartOffset.reserve((size_t)rowNum[pi]);
  }
  std::vector<uint8_t> bitmap(meta.nullMapLength);
  static const uint8_t fakeAddr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (size_t l = 0; l < n; l++) {
    int64_t p = usedRows[l];
    bool hasValidKey = (!hasFilter || filterVector[p]) && (!j.buildHasNullableKey || !nullKeyVector[p]);
    if (!hasValidKey && !keepFilteredRows) continue;
    Segment* seg = segs[partIdx[l]].get();
    if (hasValidKey) seg->validJoinKeyPos.push_back((int)seg->hashValues.size());
    seg->hashValues.push_back(hashValue[l]);
    seg->rowStartOffset.push_back(seg->rawData.size());
    int64_t rowLength = 0;
    seg->rawData.insert(seg->rawData.end(), fakeAddr, fakeAddr + 8); rowLength += 8;   // fillNextRowPtr
    if (meta.nullMapLength > 0) {   // fillNullMap :375
      std::fill(bitmap.begin(), bitmap.end(), 0);
      for (size_t ci = 0; ci < meta.rowColumnsOrder.size(); ci++) {
        int bit = (int)ci + meta.colOffsetInNullMap;
        if (col_is_null(chk.cols[meta.rowColumnsOrder[ci]], p)) bitmap[bit / 8] |= (uint8_t)(1u << (7 - bit % 8));
      }
      seg->rawData.insert(seg->rawData.end(), bitmap.begin(), bitmap.end());
      rowLength += meta.nullMapLength;
    }
    // fillSerializedKeyAndKeyLengthIfNeeded :398 (keys are fixed length here)
    if (!meta.isJoinKeysInlined) {
      if (hasValidKey) {
        seg->rawData.insert(seg->rawData.end(), keys.key(l), keys.key(l) + keys.len(l));
        rowLength += (int64_t)keys.len(l);
      } else {
        seg->rawData.insert(seg->rawData.end(), meta.fakeKeyByte.begin(), meta.fakeKeyByte.end());
        rowLength += meta.joinKeysLength;
      }
    }
    // fillRowData :433
    for (size_t ci = 0; ci < meta.rowColumnsOrder.size(); ci++) {
      const tg_column& col = chk.cols[meta.rowColumnsOrder[ci]];
      const uint8_t* r = col_raw(col, p);
      seg->rawData.insert(seg->rawData.end(), r, r + meta.columnsSize[ci]);
      rowLength += meta.columnsSize[ci];
    }
    if (rowLength % 8 != 0) seg->rawData.insert(seg->rawData.end(), fakeAddr, fakeAddr + (8 - rowLength % 8));
  }
  for (uint32_t pi = 0; pi < j.partitionNumber; pi++) {
    if (!segs[pi]->rowStartOffset.empty()) {
      segs[pi]->init_tagged_bits();
      j.rowTables[workerID][pi].push_back(std::move(segs[pi]));
    }
  }
  return true;
}

// mergeRowTablesToHashTable hash_join_v2.go:217 + buildHashTable :1458
static void build_hash_table(Join& j) {
  j.tables = std::vector<SubTable>(j.partitionNumber);
  uint8_t taggedBits = (uint8_t)kMaxTaggedBits;
  for (uint32_t pi = 0; pi < j.partitionNumber; pi++) {
    for (auto& w : j.rowTables) for (auto& seg : w[pi]) {
      j.tables[pi].segments.push_back(seg.get());
      taggedBits = std::min(taggedBits, seg->taggedBits);
    }
  }
  j.tagHelper.init(taggedBits);
  for (auto& t : j.tables) t.alloc();
  // createTasks hash_join_v2.go:1215 + checkBalance :1197: balanced (concurrency == partitions and
  // segment counts within 80% of the mean) → one whole-partition task each (non-atomic build path);
  // otherwise round-robin slices of segStep segments (CAS path, hash_table_v2.go:94).
  struct Task { uint32_t part; size_t s, e; };
  std::vector<Task> tasks;
  size_t totalSegmentCnt = 0;
  for (auto& t : j.tables) totalSegmentCnt += t.segments.size();
  bool isBalanced = j.concurrency == j.partitionNumber;
  if (isBalanced) {
    long avg = (long)(totalSegmentCnt / j.partitionNumber);
    long thr = (long)((double)avg * 0.8);
    for (auto& t : j.tables) if (std::labs((long)t.segments.size() - avg) > thr) { isBalanced = false; break; }
  }
  size_t segStep = std::max<size_t>(1, totalSegmentCnt / j.concurrency);
  if (isBalanced) {
    for (uint32_t pi = 0; pi < j.partitionNumber; pi++) tasks.push_back({pi, 0, j.tables[pi].segments.size()});
  } else {
    std::vector<size_t> start(j.partitionNumber, 0);
    for (;;) {
      bool hasNew = false;
      for (uint32_t pi = 0; pi < j.partitionNumber; pi++) {
        size_t ns = j.tables[pi].segments.size();
        if (start[pi] < ns) {
          size_t e = std::min(start[pi] + segStep, ns);
          tasks.push_back({pi, start[pi], e});
          start[pi] = e;
          hasNew = true;
        }
      }
      if (!hasNew) break;
    }
  }
  std::atomic<size_t> next{0};
  std::vector<std::thread> th;
  for (uint32_t w = 0; w < j.concurrency; w++) th.emplace_back([&] {
    for (;;) {
      size_t t = next.fetch_add(1);
      if (t >= tasks.size()) break;
      j.tables[tasks[t].part].build(tasks[t].s, tasks[t].e, j.tagHelper);
    }
  });
  for (auto& t : th) t.join();
}

// ------------------------------------------------------------------------------------------------
// probe side
// ------------------------------------------------------------------------------------------------
// isKeyMatched base_join_probe.go:820
inline bool is_key_matched(const Meta& meta, const uint8_t* key, size_t keyLen, const uint8_t* row) {
  const uint8_t* rk = row + meta.nullMapLength + sizeOfNextPtr;
  if (meta.keyMode == OneInt64) return std::memcmp(key, rk, 8) == 0;
  return std::memcmp(key, rk, keyLen) == 0;   // FixedSerializedKey: keyLen == joinKeysLength
}
// isColumnNull join_table_meta.go:105
inline bool row_col_is_null(const Meta& meta, const uint8_t* row, int columnIndex) {
  int bit = columnIndex + meta.colOffsetInNullMap;
  return (row[sizeOfNextPtr + bit / 8] & (uint8_t)(1u << (7 - bit % 8))) != 0;
}
inline void set_used_flag(uint8_t* row) {   // setUsedFlag :114 (atomic 32-bit or)
  reinterpret_cast<std::atomic<uint32_t>*>(row + sizeOfNextPtr)->fetch_or(kUsedFlagMask);
}
inline bool is_row_used(const uint8_t* row) {
  return (reinterpret_cast<const std::atomic<uint32_t>*>(row + sizeOfNextPtr)->load() & kUsedFlagMask) == kUsedFlagMask;
}

struct ProbeWorker {
  Join& j;
  std::vector<OColumn>& out;
  std::vector<int> buildUsedPosInRow;   // for each output build column: its index in rowColumnsOrder
  std::vector<int> rowColOffset;        // byte offset of each row column from rowDataOffset
  ProbeWorker(Join& jj, std::vector<OColumn>& o) : j(jj), out(o) {
    int off = 0;
    for (int sz : j.meta.columnsSize) { rowColOffset.push_back(off); off += sz; }
    for (int c : j.buildUsed) {
      int pos = -1;
      for (size_t i = 0; i < j.meta.rowColumnsOrder.size(); i++) if (j.meta.rowColumnsOrder[i] == c) pos = (int)i;
      buildUsedPosInRow.push_back(pos);
    }
  }
  // appendBuildRowToChunkInternal base_join_probe.go:589: row → columns for the used build columns
  void append_build_row(const uint8_t* row) {
    const Meta& m = j.meta;
    for (size_t k = 0; k < j.buildUsed.size(); k++) {
      OColumn& dst = out[j.buildColOffsetInResult + k];
      int pos = buildUsedPosInRow[k];
      if (m.nullMapLength > 0 && row_col_is_null(m, row, pos)) dst.append_null();
      else dst.append_raw(row + m.rowDataOffset + rowColOffset[pos]);
    }
  }
  void append_build_nulls() { for (size_t k = 0; k < j.buildUsed.size(); k++) out[j.buildColOffsetInResult + k].append_null(); }
  // appendProbeRowToChunkInternal :677 (AppendCellNTimes column.go:288)
  void append_probe_row(const tg_chunk& chk, int64_t phys, int times) {
    for (size_t k = 0; k < j.probeUsed.size(); k++) {
      const tg_column& src = chk.cols[j.probeUsed[k]];
      OColumn& dst = out[j.probeColOffsetInResult + k];
      bool isNull = col_is_null(src, phys);
      for (int t = 0; t < times; t++) { if (isNull) dst.append_null(); else dst.append_raw(col_raw(src, phys)); }
    }
  }
  void append_probe_nulls() { for (size_t k = 0; k < j.probeUsed.size(); k++) out[j.probeColOffsetInResult + k].append_null(); }
  // value of build column `col` inside a build row: false = NULL
  bool build_value(const uint8_t* row, int col, uint64_t& raw) const {
    const Meta& m = j.meta;
    int pos = -1;
    for (size_t i = 0; i < m.rowColumnsOrder.size(); i++) if (m.rowColumnsOrder[i] == col) pos = (int)i;
    if (pos < 0) return false;
    if (m.nullMapLength > 0 && row_col_is_null(m, row, pos)) return false;
    std::memcpy(&raw, row + m.rowDataOffset + rowColOffset[pos], 8);
    return true;
  }
  // OtherCondition on one candidate pair (probe row `phys` of chk, build row): every CNF item non-NULL true
  // (expression.VectorizedFilter on the joined chunk, inner_join_probe.go:72-79)
  bool other_ok(const tg_chunk& chk, int64_t phys, const uint8_t* row) const {
    for (const tg_other_item& it : j.otherCond) {
      uint64_t v[2] = {0, 0};
      for (int q = 0; q < 2; q++) {
        int side = q ? it.rhs_side : it.lhs_side, col = q ? it.rhs_col : it.lhs_col;
        if (side < 0) { if (it.is_real) std::memcpy(&v[q], &it.const_f64, 8); else v[q] = (uint64_t)it.const_i64; continue; }
        bool is_build = (side == 1) == j.rightAsBuild;
        if (is_build) { if (!build_value(row, col, v[q])) return false; }
        else { const tg_column& c = chk.cols[col]; if (col_is_null(c, phys)) return false; std::memcpy(&v[q], col_raw(c, phys), 8); }
      }
      int c;
      if (it.is_real) { double a, b; std::memcpy(&a, &v[0], 8); std::memcpy(&b, &v[1], 8); c = compare_real(a, b); }
      else c = compare_int((int64_t)v[0], it.lhs_unsigned != 0, (int64_t)v[1], it.rhs_unsigned != 0);
      bool ok;
      switch (it.op) {
        case TG_CMP_LT: ok = c < 0; break; case TG_CMP_LE: ok = c <= 0; break; case TG_CMP_GT: ok = c > 0; break;
        case TG_CMP_GE: ok = c >= 0; break; case TG_CMP_EQ: ok = c == 0; break; default: ok = c != 0; break;
      }
      if (!ok) return false;
    }
    return true;
  }

  bool process_chunk(const tg_chunk& chk) {
    // SetChunkForProbe base_join_probe.go:179
    std::vector<int64_t> usedRows; used_rows_of(chk, usedRows);
    size_t n = usedRows.size();
    if (n == 0) return true;
    int64_t physicalRows = chunk_physical_rows(chk);
    bool hasFilter = !j.probeFilter.empty();
    std::vector<uint8_t> filterVector, nullKeyVector;
    if (hasFilter) {
      filterVector.resize(physicalRows);
      for (int64_t p = 0; p < physicalRows; p++)
        filterVector[p] = filter_row(chk, p, j.probeFilter.data(), (int)j.probeFilter.size());
    }
    if (j.probeHasNullableKey) nullKeyVector.assign(physicalRows, 0);
    SerializedKeys keys;
    if (!serialize_keys(chk, j.probeKeyTypes, j.probeKeyIdx, usedRows, hasFilter ? &filterVector : nullptr,
                        j.probeHasNullableKey ? &nullKeyVector : nullptr, j.meta.serializeModes, keys))
      return false;
    std::vector<uint64_t> headers(n, 0), hashes(n, 0);
    std::vector<uint8_t> skipped(n, 0);   // filtered out or NULL key
    for (size_t l = 0; l < n; l++) {
      int64_t p = usedRows[l];
      if ((hasFilter && !filterVector[p]) || (j.probeHasNullableKey && nullKeyVector[p])) { skipped[l] = 1; continue; }
      uint64_t h = fnv1_64(keys.key(l), keys.len(l));
      hashes[l] = h;
      uint64_t part = partition_index(h, j.partitionMaskOffset);
      headers[l] = j.tables[part].lookup(h, j.tagHelper);
    }
    const Meta& meta = j.meta;
    const TagHelper& th = j.tagHelper;
    auto for_each_match = [&](size_t l, auto&& fn) {   // chain walk shared by every probe type
      uint64_t hdr = headers[l];
      while (hdr != 0) {
        uint8_t* cand = th.to_ptr(hdr);
        if (is_key_matched(meta, keys.key(l), keys.len(l), cand) && (j.otherCond.empty() || other_ok(chk, usedRows[l], cand))) { if (!fn(cand)) break; }
        hdr = next_row_address(cand, th, hashes[l]);
      }
    };
    switch (j.joinType) {
      case TG_JOIN_INNER:   // innerJoinProbe.Probe inner_join_probe.go:27
        for (size_t l = 0; l < n; l++) {
          int matched = 0;
          for_each_match(l, [&](uint8_t* row) { append_build_row(row); matched++; return true; });
          if (matched) append_probe_row(chk, usedRows[l], matched);
        }
        break;
      case TG_JOIN_LEFT_OUTER: case TG_JOIN_RIGHT_OUTER:
        if (j.needScanRowTable) {   // probeForOuterSideBuild outer_join_probe.go:308
          for (size_t l = 0; l < n; l++) {
            int matched = 0;
            for_each_match(l, [&](uint8_t* row) { append_build_row(row); set_used_flag(row); matched++; return true; });
            if (matched) append_probe_row(chk, usedRows[l], matched);
          }
        } else {                    // probeForInnerSideBuild :250 + buildResultForNotMatchedRows :229
          for (size_t l = 0; l < n; l++) {
            int matched = 0;
            for_each_match(l, [&](uint8_t* row) { append_build_row(row); matched++; return true; });
            if (matched) append_probe_row(chk, usedRows[l], matched);
            else { append_probe_row(chk, usedRows[l], 1); append_build_nulls(); }
          }
        }
        break;
      case TG_JOIN_SEMI:
        if (is_left_side_build(j)) {   // probeForLeftSideBuildNoOtherCondition semi_join_probe.go:178
          for (size_t l = 0; l < n; l++)
            for_each_match(l, [&](uint8_t* row) { if (!is_row_used(row)) set_used_flag(row); return true; });
        } else {                       // probeForRightSideBuildNoOtherCondition :262
          for (size_t l = 0; l < n; l++) {
            bool m = false;
            for_each_match(l, [&](uint8_t*) { m = true; return false; });
            if (m) append_probe_row(chk, usedRows[l], 1);
          }
        }
        break;
      case TG_JOIN_ANTI_SEMI:
        if (is_left_side_build(j)) {   // anti_semi_join_probe.go: same marking, scan emits unused rows
          for (size_t l = 0; l < n; l++)
            for_each_match(l, [&](uint8_t* row) { if (!is_row_used(row)) set_used_flag(row); return true; });
        } else {
          for (size_t l = 0; l < n; l++) {
            bool m = false;
            for_each_match(l, [&](uint8_t*) { m = true; return false; });
            if (!m) append_probe_row(chk, usedRows[l], 1);   // filtered / NULL-key probe rows are results too
          }
        }
        break;
      case TG_JOIN_LEFT_OUTER_SEMI: case TG_JOIN_ANTI_LEFT_OUTER_SEMI: {
        // left_outer_semi_join_probe.go: every probe row is emitted once with a matched flag
        bool anti = j.joinType == TG_JOIN_ANTI_LEFT_OUTER_SEMI;
        OColumn& flag = out[j.nOutCols - 1];
        for (size_t l = 0; l < n; l++) {
          bool m = false;
          for_each_match(l, [&](uint8_t*) { m = true; return false; });
          append_probe_row(chk, usedRows[l], 1);
          flag.append_i64(anti ? (m ? 0 : 1) : (m ? 1 : 0));
        }
        break;
      }
    }
    return true;
  }

  // ScanRowTable: outer_join_probe.go:117 (unused rows + NULL probe side), semi_join_probe.go:72
  // (used rows), anti_semi_join_probe.go (unused rows).  Rows [start,end) of the global row order
  // (commonInitForScanRowTable base_join_probe.go:833).
  void scan_row_table(uint64_t start, uint64_t end) {
    uint64_t idx = 0;
    for (auto& t : j.tables) for (Segment* s : t.segments) {
      for (size_t r = 0; r < s->rowStartOffset.size(); r++, idx++) {
        if (idx < start || idx >= end) continue;
        uint8_t* row = s->row_ptr(r);
        bool used = is_row_used(row);
        if (j.joinType == TG_JOIN_SEMI) { if (used) append_build_row(row); }
        else if (j.joinType == TG_JOIN_ANTI_SEMI) { if (!used) append_build_row(row); }
        else if (!used) { append_build_row(row); append_probe_nulls(); }
      }
    }
  }
};

static bool run_build(Join& j, const tg_chunk* build, int64_t nb) {
  using clk = std::chrono::steady_clock;
  uint32_t C = j.concurrency;
  j.rowTables.clear();
  j.rowTables.resize(C);
  for (auto& w : j.rowTables) w.resize(j.partitionNumber);
  auto t0 = clk::now();
  // build: fetcher → C split workers (hash_join_v2.go:1419 splitAndAppendToRowTable)
  {
    std::atomic<int64_t> next{0};
    std::atomic<bool> ok{true};
    std::vector<std::thread> th;
    for (uint32_t w = 0; w < C; w++) th.emplace_back([&, w] {
      for (;;) {
        int64_t i = next.fetch_add(1);
        if (i >= nb || !ok.load()) break;
        if (!build_process_one_chunk(j, build[i], (int)w)) ok.store(false);
      }
    });
    for (auto& t : th) t.join();
    if (!ok.load()) return false;
  }
  build_hash_table(j);
  j.buildSeconds = std::chrono::duration<double>(clk::now() - t0).count();
  return true;
}

// probe phase; may be repeated against the same built table (results are reset each time).  For joins
// that scan the row table afterwards the used flags accumulate, so repeat only inner / probe-outer joins.
static bool run_probe(Join& j, const tg_chunk* probe, int64_t np) {
  using clk = std::chrono::steady_clock;
  uint32_t C = j.concurrency;
  auto t1 = clk::now();
  // probe: C workers (hash_join_v2.go:970 runJoinWorker)
  j.results.clear();
  j.results.resize(C);
  for (auto& r : j.results) for (int el : j.outElemLen) r.emplace_back(el);
  {
    std::atomic<int64_t> next{0};
    std::atomic<bool> ok{true};
    std::vector<std::thread> th;
    for (uint32_t w = 0; w < C; w++) th.emplace_back([&, w] {
      ProbeWorker pw(j, j.results[w]);
      for (;;) {
        int64_t i = next.fetch_add(1);
        if (i >= np || !ok.load()) break;
        if (!pw.process_chunk(probe[i])) ok.store(false);
      }
    });
    for (auto& t : th) t.join();
    if (!ok.load()) return false;
  }
  if (j.needScanRowTable) {   // hash_join_v2.go:877 scanRowTableAfterProbeDone
    uint64_t total = 0;
    for (auto& t : j.tables) total += t.row_count();
    std::vector<std::thread> th;
    for (uint32_t w = 0; w < C; w++) th.emplace_back([&, w] {
      uint64_t avg = total / C, s = w * avg, e = (w == C - 1) ? total : (w + 1) * avg;
      ProbeWorker pw(j, j.results[w]);
      pw.scan_row_table(s, std::min(e, total));
    });
    for (auto& t : th) t.join();
  }
  j.probeSeconds = std::chrono::duration<double>(clk::now() - t1).count();
  return true;
}

static bool run_join(Join& j, const tg_chunk* build, int64_t nb, const tg_chunk* probe, int64_t np) {
  return run_build(j, build, nb) && run_probe(j, probe, np);
}

}  // namespace orc

// ------------------------------------------------------------------------------------------------
// C entry points
// ------------------------------------------------------------------------------------------------
using namespace orc;
struct orc_join { Join j; };

extern "C" {

uint64_t orc_fnv1_64(const uint8_t* data, size_t n) { return fnv1_64(data, n); }
uint64_t orc_next_power_of_two(uint64_t v) { return next_power_of_two(v); }
uint64_t orc_hash_table_length(uint64_t valid_keys) { return std::max<uint64_t>(next_power_of_two(valid_keys), 32); }
uint32_t orc_partition_number(uint32_t c) { return gen_partition_number(c); }
int32_t orc_partition_mask_offset(uint32_t pn) { return partition_mask_offset(pn); }
uint8_t orc_tagged_bits(uint64_t ptr) { return tagged_bits_from_ptr(ptr); }
uint64_t orc_tagged_mask(uint8_t bits) { TagHelper t; t.init(bits); return t.mask; }

static std::vector<FieldType> mk_types(int n, const int32_t* tp, const uint32_t* fl, const int32_t* bin) {
  std::vector<FieldType> v(n);
  for (int i = 0; i < n; i++) { v[i].tp = tp[i]; v[i].flag = fl ? fl[i] : 0; v[i].binary_coll = bin ? bin[i] != 0 : false; }
  return v;
}

int orc_new_table_meta(int32_t nkeys, const int32_t* build_key_index, int32_t n_build_cols,
                       const int32_t* build_types, const uint32_t* build_flags, const int32_t* build_bin,
                       const int32_t* bk_types, const uint32_t* bk_flags, const int32_t* bk_bin,
                       const int32_t* pk_types, const uint32_t* pk_flags, const int32_t* pk_bin,
                       int32_t n_other, const int32_t* other, int32_t n_output, const int32_t* output,
                       int32_t need_used_flag, orc_table_meta* out) {
  std::vector<int> ki(build_key_index, build_key_index + nkeys);
  auto bt = mk_types(n_build_cols, build_types, build_flags, build_bin);
  auto bkt = mk_types(nkeys, bk_types, bk_flags, bk_bin);
  auto pkt = mk_types(nkeys, pk_types, pk_flags, pk_bin);
  std::vector<int> ov, outv;
  if (n_other >= 0) ov.assign(other, other + n_other);
  if (n_output >= 0) outv.assign(output, output + n_output);
  Meta m = new_table_meta(ki, bt, bkt, pkt, n_other >= 0 ? &ov : nullptr, n_output >= 0 ? &outv : nullptr,
                          need_used_flag != 0);
  std::memset(out, 0, sizeof(*out));
  out->key_mode = m.keyMode; out->is_keys_inlined = m.isJoinKeysInlined;
  out->is_keys_fixed_length = m.isJoinKeysFixedLength; out->join_keys_length = m.joinKeysLength;
  out->null_map_length = m.nullMapLength; out->row_length = m.rowLength;
  out->is_fixed_length = m.isFixedLength; out->row_data_offset = m.rowDataOffset;
  out->n_row_columns = (int)m.rowColumnsOrder.size();
  for (size_t i = 0; i < m.rowColumnsOrder.size() && i < 64; i++) out->row_columns_order[i] = m.rowColumnsOrder[i];
  out->n_serialize_modes = (int)m.serializeModes.size();
  for (size_t i = 0; i < m.serializeModes.size() && i < 16; i++) out->serialize_modes[i] = m.serializeModes[i];
  out->column_count_needed_for_other_condition = m.columnCountNeededForOtherCondition;
  return 0;
}

int orc_join_open(const tg_join_desc* d, int32_t concurrency, orc_join** out) {
  auto* h = new orc_join();
  Join& j = h->j;
  j.joinType = d->join_type; j.rightAsBuild = d->build_is_right != 0;
  j.leftTypes = mk_types(d->n_left_cols, d->left_types, d->left_flags, nullptr);
  j.rightTypes = mk_types(d->n_right_cols, d->right_types, d->right_flags, nullptr);
  j.leftKeyIdx.assign(d->left_key_idx, d->left_key_idx + d->nkeys);
  j.rightKeyIdx.assign(d->right_key_idx, d->right_key_idx + d->nkeys);
  if (d->n_lused < 0) for (int i = 0; i < d->n_left_cols; i++) j.lUsed.push_back(i);
  else j.lUsed.assign(d->lused, d->lused + d->n_lused);
  if (d->n_rused < 0) for (int i = 0; i < d->n_right_cols; i++) j.rUsed.push_back(i);
  else j.rUsed.assign(d->rused, d->rused + d->n_rused);
  if (d->n_build_filter > 0) j.buildFilter.assign(d->build_filter, d->build_filter + d->n_build_filter);
  if (d->n_probe_filter > 0) j.probeFilter.assign(d->probe_filter, d->probe_filter + d->n_probe_filter);
  if (d->n_other_cond > 0 && d->other_cond) j.otherCond.assign(d->other_cond, d->other_cond + d->n_other_cond);
  j.concurrency = (uint32_t)std::max(1, concurrency);
  std::string err;
  if (!setup_join(j, err)) { set_error(err); delete h; return TG_ERR_UNSUPPORTED; }
  *out = h;
  return 0;
}

int orc_join_run(orc_join* h, const tg_chunk* b, int64_t nb, const tg_chunk* p, int64_t np) {
  return run_join(h->j, b, nb, p, np) ? 0 : TG_ERR_UNSUPPORTED;
}
int orc_join_build(orc_join* h, const tg_chunk* b, int64_t nb) { return run_build(h->j, b, nb) ? 0 : TG_ERR_UNSUPPORTED; }
int orc_join_probe(orc_join* h, const tg_chunk* p, int64_t np) { return run_probe(h->j, p, np) ? 0 : TG_ERR_UNSUPPORTED; }
int64_t orc_join_result_rows(orc_join* h) {
  int64_t n = 0;
  for (auto& r : h->j.results) if (!r.empty()) n += r[0].length;
  return n;
}
int32_t orc_join_result_cols(orc_join* h) { return h->j.nOutCols; }
int orc_join_result_fetch(orc_join* h, tg_mut_chunk* out) {
  std::vector<std::vector<OColumn>*> parts;
  for (auto& r : h->j.results) parts.push_back(&r);
  return fetch_result(parts, h->j.nOutCols, out);
}
int64_t orc_join_row_count(orc_join* h) { int64_t n = 0; for (auto& t : h->j.tables) n += (int64_t)t.row_count(); return n; }
int64_t orc_join_total_row_bytes(orc_join* h) {
  int64_t n = 0;
  for (auto& t : h->j.tables) for (auto* s : t.segments) n += (int64_t)s->rawData.size();
  return n;
}
int64_t orc_join_hash_table_slots(orc_join* h) { int64_t n = 0; for (auto& t : h->j.tables) n += (int64_t)t.hashTable.size(); return n; }
int32_t orc_join_partitions(orc_join* h) { return (int32_t)h->j.partitionNumber; }
double orc_join_build_seconds(orc_join* h) { return h->j.buildSeconds; }
double orc_join_probe_seconds(orc_join* h) { return h->j.probeSeconds; }
void orc_join_close(orc_join* h) { delete h; }

}  // extern "C"
