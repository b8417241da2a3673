// amgpu — columns with ids this version does not know (written by a future version of Automerge): carried through apply,
// save and load like the reference does (new.js:1406-1424 updateBlockColumns; readOperation new.js:570-610 reads them by
// column TYPE: id & 7). They never influence the op set or the patches, and real documents do not have them, so this is
// host code off the hot path: the decode kernel only raises a flag when it meets an unknown column id; the host then
// decodes those columns of the applied changes with the same readers the kernels use (decode.cuh, HD functions), keeps the
// values per op id, and save() encodes them into document columns in document order (canonical RLE / delta / boolean forms
// of encoding.js:558-783, 932-998, 1061-1135).
#pragma once
#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>
#include "doccols.cuh"

namespace amg {

struct UnknownValue { bool isNull = true; long long num = 0; std::string bytes; };   // number (uint / int / delta / boolean) or bytes (utf8 / raw)
typedef std::map<u32, std::vector<UnknownValue>> UnknownRow;                          // column id -> the op's values in that column

struct UnknownStore {
  std::unordered_map<u64, UnknownRow> byOp;   // packed op id -> its values
  std::set<u32> colIds;
  bool empty() const { return colIds.empty(); }
  void clear() { byOp.clear(); colIds.clear(); }
};

inline bool is_known_change_column(u32 id) { return col_index_of(id) >= 0; }
// an op column of the document format, or one of the change format's (a pred column in a document is skipped, not carried)
inline bool is_known_doc_column(u32 id) { return std::count(DOC_COL_IDS, DOC_COL_IDS + NUM_DOC_COLS, id) > 0 || is_known_change_column(id); }

// one value-at-a-time reader for a column of any type (what makeDecoders gives readOperation)
struct AnyColumnReader {
  u32 id; int type; RleReader rle; ByteReader raw; bool bval = true, bfirst = true; u64 bcount = 0; long long acc = 0;
  AnyColumnReader(const u8* base, u32 id_, u32 off, u32 len) : id(id_), type((int)(id_ & 7)), rle(base, off, off + len, (id_ & 7) == 5 ? 2 : ((id_ & 7) == 3 ? 1 : 0)), raw(base, off, off + len) {}
  // GROUP_CARD / ACTOR_ID / INT_RLE / VALUE_LEN: uint; INT_DELTA: running sum; BOOLEAN; STRING_RLE
  u32 read(UnknownValue& v) {
    v = UnknownValue();
    if (type == 4) {
      bool out = false;
      if (!(bcount == 0 && raw.done())) {
        while (bcount == 0) { bcount = raw.uleb(); bval = !bval; if (raw.err) return raw.err; if (bcount == 0 && !bfirst) return KE_BOOL_ZERO; bfirst = false; }
        bcount--; out = bval;
      }
      v.isNull = false; v.num = out ? 1 : 0; return 0;
    }
    long long n = 0; u32 o = 0, l = 0; const bool nn = rle.next(n, o, l);
    if (rle.r.err) return rle.r.err;
    if (!nn) return 0;
    v.isNull = false;
    if (type == 5) v.bytes.assign((const char*)rle.r.src.base + o, l);
    else if (type == 3) { acc += n; v.num = acc; }
    else v.num = n;
    return 0;
  }
  u32 readRaw(u64 n, UnknownValue& v) { v = UnknownValue(); if ((u64)raw.pos + n > raw.end) return KE_SUBARRAY; v.isNull = false; v.bytes.assign((const char*)raw.src.base + raw.pos, (size_t)n); raw.pos += (u32)n; return 0; }
};

// readOperation (new.js:570-610) over every column of a change / document in directory order; calls sink(opIndex, row) with
// the values of the unknown columns. `cols`: (id, offset, length) ascending; numOps rows are read.
template <class Known, class Sink> inline u32 read_unknown_columns(const u8* base, const std::vector<std::array<u32, 3>>& cols, size_t numOps, Known isKnown, Sink sink) {
  std::vector<AnyColumnReader> readers; for (auto& c : cols) readers.emplace_back(base, c[0], c[1], c[2]);
  for (size_t i = 0; i < numOps; i++) {
    UnknownRow row; long long lastGroup = -1; u64 card = 0; long long valueColumn = -1; u64 valueBytes = 0;
    for (auto& r : readers) {
      const bool keep = !isKnown(r.id); std::vector<UnknownValue> vals; UnknownValue v; u32 e = 0;
      if (r.type == 7) {                                               // VALUE_RAW
        if ((long long)r.id != valueColumn) return KE_UNSUPPORTED_OP;  // "unexpected VALUE_RAW column"
        e = r.readRaw(valueBytes, v); vals.push_back(v);
      } else if (r.type == 0) {                                        // GROUP_CARD
        lastGroup = r.id >> 4; e = r.read(v); card = v.isNull ? 0 : (u64)v.num;
        if (v.isNull) { v.isNull = false; v.num = 0; }   // `readValue() || 0` (new.js:581): a missing cardinality is written back as 0
        vals.push_back(v);
      } else if ((long long)(r.id >> 4) == lastGroup) {
        if (r.type == 6) { valueColumn = r.id + 1; valueBytes = 0; }
        for (u64 k = 0; k < card && !e; k++) { e = r.read(v); if (r.type == 6 && !v.isNull) valueBytes += (u64)v.num >> 4; vals.push_back(v); }
      } else {
        e = r.read(v); if (r.type == 6) { valueColumn = r.id + 1; valueBytes = v.isNull ? 0 : ((u64)v.num >> 4); } vals.push_back(v);
      }
      if (e) return e;
      if (keep) row[r.id] = std::move(vals);
    }
    sink(i, row);
  }
  return 0;
}

// ---- canonical column encoders (host): encoding.js:558-783 RLEEncoder, 932-998 DeltaEncoder, 1061-1135 BooleanEncoder
inline void put_uleb(std::string& o, u64 v) { do { u8 b = v & 0x7f; v >>= 7; if (v) b |= 0x80; o.push_back((char)b); } while (v); }
inline void put_sleb(std::string& o, long long v) { while (true) { u8 b = v & 0x7f; v >>= 7; if ((v == 0 && !(b & 0x40)) || (v == -1 && (b & 0x40))) { o.push_back((char)b); return; } o.push_back((char)(b | 0x80)); } }
inline std::string encode_rle_column(const std::vector<UnknownValue>& vals, int kind /* 0 uint, 1 int, 2 utf8 */) {
  bool allNull = true; for (auto& v : vals) if (!v.isNull) { allNull = false; break; }
  std::string out; if (allNull) return out;
  auto same = [&](const UnknownValue& a, const UnknownValue& b) { return a.isNull == b.isNull && (a.isNull || (kind == 2 ? a.bytes == b.bytes : a.num == b.num)); };
  auto putRaw = [&](const UnknownValue& v) { if (kind == 0) put_uleb(out, (u64)v.num); else if (kind == 1) put_sleb(out, v.num); else { put_uleb(out, v.bytes.size()); out += v.bytes; } };
  std::vector<const UnknownValue*> lit;
  auto flush = [&]() { if (lit.empty()) return; put_sleb(out, -(long long)lit.size()); for (auto* x : lit) putRaw(*x); lit.clear(); };
  for (size_t i = 0; i < vals.size();) {
    size_t j = i + 1; while (j < vals.size() && same(vals[i], vals[j])) j++;
    const size_t n = j - i;
    if (vals[i].isNull) { flush(); put_sleb(out, 0); put_uleb(out, n); }
    else if (n >= 2) { flush(); put_sleb(out, (long long)n); putRaw(vals[i]); }
    else lit.push_back(&vals[i]);
    i = j;
  }
  flush();
  return out;
}
inline std::string encode_delta_column(const std::vector<UnknownValue>& vals) {
  std::vector<UnknownValue> d(vals.size()); long long last = 0;
  for (size_t i = 0; i < vals.size(); i++) { d[i].isNull = vals[i].isNull; if (!vals[i].isNull) { d[i].num = vals[i].num - last; last = vals[i].num; } }
  return encode_rle_column(d, 1);
}
inline std::string encode_bool_column(const std::vector<UnknownValue>& vals) {
  std::string out; bool last = false; u64 count = 0;
  for (auto& v : vals) { const bool b = !v.isNull && v.num != 0; if (b == last) count++; else { put_uleb(out, count); last = b; count = 1; } }
  if (count > 0) put_uleb(out, count);
  return out;
}
inline std::string encode_unknown_column(u32 id, const std::vector<UnknownValue>& vals) {
  switch (id & 7) {
    case 3: return encode_delta_column(vals);
    case 4: return encode_bool_column(vals);
    case 5: return encode_rle_column(vals, 2);
    case 7: { std::string out; for (auto& v : vals) out += v.bytes; return out; }
    default: return encode_rle_column(vals, 0);
  }
}

}  // namespace amg
