// amgpu — parallel decode of long RLE / delta / boolean columns (the columns of a saved document hold one value per op or
// per change of the whole history: 10^6 values in one byte stream).
//
// Replaces, for long columns (reference paths relative to /root/reference):
//   backend/encoding.js:789-920   RLEDecoder   (count / value records)
//   backend/encoding.js:1004-1051 DeltaDecoder (prefix sum over an RLE column of differences)
//   backend/encoding.js:1141-1207 BooleanDecoder (alternating run lengths)
// as used by the document load path (backend/new.js:1695-1750, columnar.js:1006-1038).
//
// A byte stream of LEB128 numbers has no random access, but it has two parallel handles:
//   1. tokens: a number ends at every byte whose top bit is clear - one flag per byte, one prefix sum, and every
//      token knows its index and its first byte; all tokens are decoded at once;
//   2. records: whether a token is a record head (count) or a value depends on everything before it, but "if token t is
//      a head, the next head is t + 2 (repetition, null run) or t + 1 + n (literal run of n)" is known for every token on
//      its own. The heads are the tokens reachable from token 0 along that successor function: pointer doubling,
//      ceil(log2 T) rounds.
// Then records -> value counts -> prefix sum -> one thread per output value.
//
// This path only accepts streams in the canonical form the reference's encoders produce and its decoders insist on,
// holding exactly the expected number of values. Anything else (malformed, short, over-long, numbers beyond 53 bits)
// makes it return false, and the caller runs the serial decoder (decode_one_column / LoadedColKernel), which is the one
// that reports errors the way the reference does. utf8 columns (keyStr, message) always take the serial decoder.
#pragma once
#include "encode.cuh"
#include "prims.cuh"

namespace amg {

struct PcTokEndKernel { const u8* bytes; u32* flag; HD void operator()(size_t p) const { flag[p] = (bytes[p] & 0x80) ? 0u : 1u; } };
struct PcTokStartKernel {   // token index of a byte = number of token ends before it
  const u32* flag; const u32* endsBefore; u32* tokPos;
  HD void operator()(size_t p) const { if (p == 0 || flag[p - 1]) tokPos[endsBefore[p]] = (u32)p; }
};
// value of every token under both readings (unsigned LEB128 / signed LEB128). Numbers of more than 8 bytes (56 bits) are
// beyond the 53-bit range of the format or non-minimal: not handled here (bad).
struct PcTokValueKernel {
  const u8* bytes; const u32* tokPos; u32 numBytes; u32 T; u64* tokU; long long* tokS; u32* bad;
  HD void operator()(size_t t) const {
    const u32 p0 = tokPos[t], p1 = t + 1 < T ? tokPos[t + 1] : numBytes; const u32 nb = p1 - p0;
    if (nb > 8) { *bad = 1; tokU[t] = 0; tokS[t] = 0; return; }
    u64 u = 0; for (u32 i = 0; i < nb; i++) u |= (u64)(bytes[p0 + i] & 0x7f) << (7 * i);
    tokU[t] = u;
    long long s = (long long)u; if (bytes[p1 - 1] & 0x40) s |= (long long)(~0ULL << (7 * nb));
    tokS[t] = s;
  }
};
// successor of token t if t is a record head; defects of the record are kept per token and only matter if t is reached
struct PcNextKernel {
  const long long* tokS; const u64* tokU; u32 T; u32* nxt; u32* defect;
  HD void operator()(size_t t) const {
    if (t == T) { nxt[t] = T; defect[t] = 0; return; }
    const long long c = tokS[t]; u64 n; u32 d = 0;
    if (c > 1) n = t + 2;
    else if (c == 1) { n = t + 2; d = 1; }                       // "Repetition count of 1 is not allowed"
    else if (c < 0) n = (u64)t + 1 + (u64)(-c);
    else { n = t + 2; if (t + 1 >= T || tokU[t + 1] == 0) d = 1; }   // "Zero-length null runs are not allowed"
    if (n > T) { n = T; d = 1; }                                  // record runs past the end of the column
    nxt[t] = (u32)n; defect[t] = d;
  }
};
struct PcReachRoundKernel {   // after round r every head at distance < 2^(r+1) from token 0 is marked
  u32* reach; const u32* jumpIn; u32* jumpOut;
  HD void operator()(size_t t) const { const u32 j = jumpIn[t]; if (reach[t]) reach[j] = 1; jumpOut[t] = jumpIn[j]; }
};
struct PcHeadFlagKernel { const u32* reach; const u32* defect; u32 T; u32* head; u32* bad; HD void operator()(size_t t) const { const u32 h = (t < T && reach[t]) ? 1u : 0u; head[t] = h; if (h && defect[t]) *bad = 1; } };
enum { PC_REP = 0, PC_LIT = 1, PC_NULL = 2 };
struct PcRecordKernel {   // one entry per record: head token, kind, number of values
  const u32* head; const u32* recIdx; const long long* tokS; const u64* tokU; u32 T; u32* recTok; u32* recN; u32* bad;
  HD void operator()(size_t t) const {
    if (!head[t]) return;
    const u32 r = recIdx[t]; recTok[r] = (u32)t;
    const long long c = tokS[t]; u64 n = c > 1 ? (u64)c : (c < 0 ? (u64)(-c) : tokU[t + 1]);
    if (n > 0x7fffffffULL) { *bad = 1; n = 0; }
    recN[r] = (u32)n;
  }
};
HD u32 pc_record_of(const u32* recOff, u32 R, u32 i) {   // last r with recOff[r] <= i (recOff is non-decreasing, recOff[R] = total)
  u32 lo = 0, hi = R;
  while (hi - lo > 1) { const u32 mid = (lo + hi) >> 1; if (recOff[mid] <= i) lo = mid; else hi = mid; }
  return lo;
}
// One thread per value. Also insists on the canonical form: no equal neighbours except inside a repetition, no literal
// after a literal, no null run after a null run (encoding.js:865-887 / 536-557).
struct PcExpandKernel {
  const u32* recTok; const u32* recOff; u32 R; const long long* tokS; const u64* tokU; int isSigned; long long* vals; u32* bad;
  HD int kindOf(u32 r) const { const long long c = tokS[recTok[r]]; return c > 1 ? PC_REP : (c < 0 ? PC_LIT : PC_NULL); }
  HD long long value(u32 tok) const {
    if (isSigned) { const long long s = tokS[tok]; if (s < -((1LL << 53) - 1) || s > ((1LL << 53) - 1)) *bad = 1; return s; }
    const u64 u = tokU[tok]; if (u > ((1ULL << 53) - 1)) *bad = 1; return (long long)u;
  }
  HD void operator()(size_t i) const {
    const u32 r = pc_record_of(recOff, R, (u32)i); const u32 t = recTok[r]; const int kind = kindOf(r); const u32 k = (u32)i - recOff[r];
    long long v = NULLV;
    if (kind == PC_REP) v = value(t + 1); else if (kind == PC_LIT) v = value(t + 1 + k);
    vals[i] = v;
    if (kind == PC_LIT && k > 0) { if (value(t + k) == v) *bad = 1; }   // repetition inside a literal run
    if (k == 0 && r > 0) {   // first value of a record against the record before it
      const int pk = kindOf(r - 1); const u32 pt = recTok[r - 1];
      if (pk == PC_NULL && kind == PC_NULL) *bad = 1;
      if (pk == PC_LIT && kind == PC_LIT) *bad = 1;
      if (pk != PC_NULL && kind != PC_NULL) { const long long pv = pk == PC_REP ? value(pt + 1) : value(pt + (recOff[r] - recOff[r - 1])); if (pv == v) *bad = 1; }
    }
  }
};

// ---- consumers of the decoded int64 values
struct PcToU32Kernel { const long long* v; u32* out; u32* bad; HD void operator()(size_t i) const { const long long x = v[i]; if (x == NULLV) { out[i] = NULL32; return; } if ((u64)x > 0xfffffffeULL) { *bad = 1; out[i] = 0; return; } out[i] = (u32)x; } };
struct PcDeltaInput { const long long* v; HD u64 operator()(size_t i) const { return v[i] == NULLV ? 0ull : (u64)v[i]; } };
struct PcDeltaToU32Kernel {   // running sum of the differences (nulls do not move it and stay null); the values must fit the u32 row fields
  const long long* v; const u64* excl; u32* out; u32* bad;
  HD void operator()(size_t i) const {
    if (v[i] == NULLV) { out[i] = NULL32; return; }
    const long long acc = (long long)(excl[i] + (u64)v[i]);
    if (acc < 0 || acc > 0xfffffffeLL) { *bad = 1; out[i] = 0; return; }
    out[i] = (u32)acc;
  }
};
struct PcDeltaToI64Kernel { const long long* v; const u64* excl; long long* out; HD void operator()(size_t i) const { out[i] = v[i] == NULLV ? NULLV : (long long)(excl[i] + (u64)v[i]); } };
struct PcLenBytesKernel { const long long* v; u32* bytes; u32* bad; HD void operator()(size_t i) const { const long long x = v[i]; u64 b = x == NULLV ? 0 : ((u64)x >> 4); if (b > 0x7fffffffULL) { *bad = 1; b = 0; } bytes[i] = (u32)b; } };
struct PcCountKernel { const long long* v; u32* cnt; u32* bad; HD void operator()(size_t i) const { const long long x = v[i]; u64 c = x == NULLV ? 0 : (u64)x; if (c > 0x7fffffffULL) { *bad = 1; c = 0; } cnt[i] = (u32)c; } };
struct PcAddBaseKernel { u32* a; u32 base; HD void operator()(size_t i) const { a[i] += base; } };
struct PcCopyI64Kernel { const long long* in; long long* out; HD void operator()(size_t i) const { out[i] = in[i]; } };

// ---- boolean columns: the tokens are run lengths, values alternate starting with false
struct PcBoolRunKernel { const u64* tokU; u32* runLen; u32* bad; HD void operator()(size_t t) const { const u64 n = tokU[t]; if ((n == 0 && t > 0) || n > 0x7fffffffULL) { *bad = 1; runLen[t] = 0; return; } runLen[t] = (u32)n; } };
struct PcBoolExpandKernel {   // a reader past the end of the column yields false
  const u32* runOff; u32 T; u32* out;
  HD void operator()(size_t i) const { if ((u32)i >= runOff[T]) { out[i] = 0; return; } out[i] = pc_record_of(runOff, T, (u32)i) & 1u; }
};

// Parallel decoder kinds (ParColumnDecoder::decode). Values go to the row field `u` (NULL32 for null) or, where there is
// none, to `v` (NULLV for null); PK_LEN / PK_COUNT / PK_EXTRA_LEN also write the running offsets and the total.
enum ParKind { PK_NONE, PK_UINT, PK_INT, PK_DELTA, PK_BOOL, PK_LEN, PK_COUNT, PK_EXTRA_LEN };
struct PcOut { u32* u = nullptr; long long* v = nullptr; u32* off = nullptr; u32* len = nullptr; u32 base = 0; u64* sum = nullptr; };

struct ParColumnDecoder {
  Ctx& ctx; ScanTemp& st;
  DBuf<u32> flag, ends, tokPos, nxtA, nxtB, reach, defect, recIdx, recTok, recN, recOff, word; DBuf<u64> tokU, excl; DBuf<long long> tokS, vals;
  size_t numTokens = 0;
  ParColumnDecoder(Ctx& c, ScanTemp& s) : ctx(c), st(s) {}
  u32 readU32(const u32* p) { u32 v = 0; d2h(ctx, &v, p, 4); sync(ctx); return v; }
  // tokens of bytes[0, len): false if the stream ends inside a number or holds a number this path does not take
  bool tokenize(const u8* bytes, size_t len) {
    flag.ensure(ctx, len + 1); ends.ensure(ctx, len + 2); word.ensure(ctx, 4); dev_memset(ctx, word.p, 0, 16);
    foreach(ctx, len, PcTokEndKernel{bytes, flag.p});
    scan_exclusive(ctx, st, flag.p, ends.p, len);
    u32 lastFlag = 0, T = 0; d2h(ctx, &lastFlag, flag.p + len - 1, 4); d2h(ctx, &T, ends.p + len, 4); sync(ctx);
    if (!lastFlag) return false;
    numTokens = T;
    tokPos.ensure(ctx, T + 2); tokU.ensure(ctx, T + 2); tokS.ensure(ctx, T + 2);
    foreach(ctx, len, PcTokStartKernel{flag.p, ends.p, tokPos.p});
    foreach(ctx, T, PcTokValueKernel{bytes, tokPos.p, (u32)len, T, tokU.p, tokS.p, word.p});
    dev_memset(ctx, tokU.p + T, 0, 16); dev_memset(ctx, tokS.p + T, 0, 16);
    return true;
  }
  size_t numRecords = 0;
  // RLE column of numbers holding exactly n values -> vals[0, n) (NULLV = null). false: take the serial decoder.
  bool rle(const u8* bytes, size_t len, bool isSigned, size_t n) {
    u32 total = 0;
    if (n == 0 || !rleRecords(bytes, len, &total) || total != n) return false;
    vals.ensure(ctx, n + 1);
    foreach(ctx, n, PcExpandKernel{recTok.p, recOff.p, (u32)numRecords, tokS.p, tokU.p, isSigned ? 1 : 0, vals.p, word.p});
    return readU32(word.p) == 0;
  }
  // records of an RLE column of numbers and the number of values they stand for
  bool rleRecords(const u8* bytes, size_t len, u32* totalOut) {
    if (len == 0 || len >= 0x7fffffffULL) return false;
    if (!tokenize(bytes, len)) return false;
    const u32 T = (u32)numTokens;
    nxtA.ensure(ctx, T + 2); nxtB.ensure(ctx, T + 2); reach.ensure(ctx, T + 2); defect.ensure(ctx, T + 2);
    foreach(ctx, (size_t)T + 1, PcNextKernel{tokS.p, tokU.p, T, nxtA.p, defect.p});
    dev_memset(ctx, reach.p, 0, ((size_t)T + 1) * 4); fill32(reach.p, 1, 1);
    u32* a = nxtA.p; u32* b = nxtB.p;
    for (u32 span = 1; span < T + 1; span <<= 1) { foreach(ctx, (size_t)T + 1, PcReachRoundKernel{reach.p, a, b}); std::swap(a, b); }
    recIdx.ensure(ctx, T + 3);
    u32* head = nxtA.p == a ? nxtB.p : nxtA.p;   // the jump table that is not current is free
    foreach(ctx, (size_t)T + 1, PcHeadFlagKernel{reach.p, defect.p, T, head, word.p});
    scan_exclusive(ctx, st, head, recIdx.p, (size_t)T + 1);
    u32 R = 0, endReached = 0, bad = 0; d2h(ctx, &R, recIdx.p + T + 1, 4); d2h(ctx, &endReached, reach.p + T, 4); d2h(ctx, &bad, word.p, 4); sync(ctx);
    if (bad || !endReached || R == 0) return false;
    recTok.ensure(ctx, R + 2); recN.ensure(ctx, R + 2); recOff.ensure(ctx, R + 3);
    foreach(ctx, T, PcRecordKernel{head, recIdx.p, tokS.p, tokU.p, T, recTok.p, recN.p, word.p});
    scan_exclusive(ctx, st, recN.p, recOff.p, R);
    excl.ensure(ctx, (size_t)R + 2); scan_exclusive64(ctx, st, PcDeltaInputU32{recN.p}, excl.p, R);   // 64-bit total: the 32-bit offsets must not have wrapped
    u64 last = 0; u32 lastN = 0; d2h(ctx, &last, excl.p + R - 1, 8); d2h(ctx, &lastN, recN.p + R - 1, 4); d2h(ctx, &bad, word.p, 4); sync(ctx);
    if (bad || last + lastN > 0x7ffffffeULL) return false;
    numRecords = R; *totalOut = (u32)(last + lastN);
    return true;
  }
  void fill32(u32* p, u32 v, size_t n) { std::vector<u32> h(n, v); h2d(ctx, p, h.data(), n * 4); sync(ctx); }
  bool checkBad() { return readU32(word.p) == 0; }
  // ---- typed outputs (each returns false like rle())
  bool toU32(const u8* bytes, size_t len, size_t n, u32* out) { if (!rle(bytes, len, false, n)) return false; foreach(ctx, n, PcToU32Kernel{vals.p, out, word.p}); return checkBad(); }
  bool deltaToU32(const u8* bytes, size_t len, size_t n, u32* out) {
    if (!rle(bytes, len, true, n)) return false;
    excl.ensure(ctx, n + 2); scan_exclusive64(ctx, st, PcDeltaInput{vals.p}, excl.p, n);
    foreach(ctx, n, PcDeltaToU32Kernel{vals.p, excl.p, out, word.p}); return checkBad();
  }
  bool toI64(const u8* bytes, size_t len, bool isSigned, size_t n, long long* out) { if (!rle(bytes, len, isSigned, n)) return false; foreach(ctx, n, PcCopyI64Kernel{vals.p, out}); return true; }
  bool deltaToI64(const u8* bytes, size_t len, size_t n, long long* out) {
    if (!rle(bytes, len, true, n)) return false;
    excl.ensure(ctx, n + 2); scan_exclusive64(ctx, st, PcDeltaInput{vals.p}, excl.p, n);
    foreach(ctx, n, PcDeltaToI64Kernel{vals.p, excl.p, out}); return true;
  }
  // valLen-style column: out = value (NULL32 for null), off = base + running sum of (value >> 4); *sumOut = that sum
  bool lenColumn(const u8* bytes, size_t len, size_t n, u32* out, u32* off, u32 base, u64* sumOut) {
    if (!rle(bytes, len, false, n)) return false;
    foreach(ctx, n, PcToU32Kernel{vals.p, out, word.p});
    recN.ensure(ctx, n + 2); recOff.ensure(ctx, n + 3);
    foreach(ctx, n, PcLenBytesKernel{vals.p, recN.p, word.p});
    scan_exclusive(ctx, st, recN.p, recOff.p, n);
    excl.ensure(ctx, n + 2); scan_exclusive64(ctx, st, PcDeltaInputU32{recN.p}, excl.p, n);   // 64-bit total: the 32-bit running sum must not have wrapped
    u64 last = 0; u32 lastN = 0; d2h(ctx, &last, excl.p + n - 1, 8); d2h(ctx, &lastN, recN.p + n - 1, 4); sync(ctx);
    *sumOut = last + lastN; if (*sumOut > 0x7fffffffULL) return false;
    d2d(ctx, off, recOff.p, n * 4); if (base) foreach(ctx, n, PcAddBaseKernel{off, base});
    return checkBad();
  }
  struct PcDeltaInputU32 { const u32* v; HD u64 operator()(size_t i) const { return v[i]; } };
  // predNum-style column: cnt = value (0 for null), off = running sum of the counts; *sumOut = total
  bool countColumn(const u8* bytes, size_t len, size_t n, u32* cnt, u32* off, u64* sumOut) {
    if (!rle(bytes, len, false, n)) return false;
    foreach(ctx, n, PcCountKernel{vals.p, cnt, word.p});
    recOff.ensure(ctx, n + 3); scan_exclusive(ctx, st, cnt, recOff.p, n);
    excl.ensure(ctx, n + 2); scan_exclusive64(ctx, st, PcDeltaInputU32{cnt}, excl.p, n);
    u64 last = 0; u32 lastN = 0; d2h(ctx, &last, excl.p + n - 1, 8); d2h(ctx, &lastN, cnt + n - 1, 4); sync(ctx);
    *sumOut = last + lastN; if (*sumOut > 0x7fffffffULL) return false;
    d2d(ctx, off, recOff.p, n * 4);
    return checkBad();
  }
  // extraLen-style column of the change metadata: out = value (NULLV for null), strLen = value >> 4, strOff = base + running sum of those
  bool extraLenColumn(const u8* bytes, size_t len, size_t n, long long* out, u32* strOff, u32* strLen, u32 base) {
    if (!rle(bytes, len, false, n)) return false;
    foreach(ctx, n, PcCopyI64Kernel{vals.p, out});
    recOff.ensure(ctx, n + 3);
    foreach(ctx, n, PcLenBytesKernel{vals.p, strLen, word.p});
    scan_exclusive(ctx, st, strLen, recOff.p, n);
    excl.ensure(ctx, n + 2); scan_exclusive64(ctx, st, PcDeltaInputU32{strLen}, excl.p, n);
    u64 last = 0; u32 lastN = 0; d2h(ctx, &last, excl.p + n - 1, 8); d2h(ctx, &lastN, strLen + n - 1, 4); sync(ctx);
    if (last + lastN + base > 0x7fffffffULL) return false;
    d2d(ctx, strOff, recOff.p, n * 4); if (base) foreach(ctx, n, PcAddBaseKernel{strOff, base});
    return checkBad();
  }
  // sum of the n values of a column of counts (nulls count as 0)
  bool sumColumn(const u8* bytes, size_t len, size_t n, u64* sumOut) {
    if (!rle(bytes, len, false, n)) return false;
    excl.ensure(ctx, n + 2); scan_exclusive64(ctx, st, PcDeltaInput{vals.p}, excl.p, n);
    u64 last = 0; long long lastV = 0; d2h(ctx, &last, excl.p + n - 1, 8); d2h(ctx, &lastV, vals.p + n - 1, 8); sync(ctx);
    *sumOut = last + (lastV == NULLV ? 0ull : (u64)lastV);
    return true;
  }
  bool boolean(const u8* bytes, size_t len, size_t n, u32* out) {
    if (len == 0 || n == 0 || len >= 0x7fffffffULL) return false;
    if (!tokenize(bytes, len)) return false;
    const u32 T = (u32)numTokens;
    recN.ensure(ctx, T + 2); recOff.ensure(ctx, T + 3);
    foreach(ctx, T, PcBoolRunKernel{tokU.p, recN.p, word.p});
    scan_exclusive(ctx, st, recN.p, recOff.p, T);
    excl.ensure(ctx, T + 2); scan_exclusive64(ctx, st, PcDeltaInputU32{recN.p}, excl.p, T);
    u64 last = 0; u32 lastN = 0; d2h(ctx, &last, excl.p + T - 1, 8); d2h(ctx, &lastN, recN.p + T - 1, 4); sync(ctx);
    if (last + lastN > 0x7fffffffULL || last + lastN < n) return false;   // (a column shorter than its rows is legal, but what a reader does at its end depends on the last run: serial)
    if (!checkBad()) return false;
    foreach(ctx, n, PcBoolExpandKernel{recOff.p, T, out});
    return true;
  }
  // n values of one column through the decoder of its kind (false: take the serial decoder)
  bool decode(int kind, const u8* bytes, size_t len, size_t n, const PcOut& o) {
    switch (kind) {
      case PK_UINT: return o.u ? toU32(bytes, len, n, o.u) : toI64(bytes, len, false, n, o.v);
      case PK_INT: return toI64(bytes, len, true, n, o.v);
      case PK_DELTA: return o.u ? deltaToU32(bytes, len, n, o.u) : deltaToI64(bytes, len, n, o.v);
      case PK_BOOL: return boolean(bytes, len, n, o.u);
      case PK_LEN: return lenColumn(bytes, len, n, o.u, o.off, o.base, o.sum);
      case PK_COUNT: return countColumn(bytes, len, n, o.u, o.off, o.sum);
      case PK_EXTRA_LEN: return extraLenColumn(bytes, len, n, o.v, o.off, o.len, o.base);
      default: return false;   // utf8 and raw bytes: serial only
    }
  }
};

// The parallel decoder of each change column kind (utf8, raw bytes, child columns: none) and the row fields it fills
// (rows of one change start at rowBase, its preds at predBase; valBase: arena offset of its valRaw column).
static const int CX_PAR_KIND[NCOLS] = {PK_UINT, PK_UINT, PK_UINT, PK_DELTA, PK_NONE, PK_BOOL, PK_UINT, PK_LEN, PK_NONE, PK_NONE, PK_NONE, PK_COUNT, PK_UINT, PK_DELTA};
inline PcOut cx_outputs(const RawRows& r, int cx, u32 rowBase, u32 predBase, u32 valBase, u64* sum) {
  u32* const field[NCOLS] = {r.objActor, r.objCtr, r.keyActor, r.keyCtr, nullptr, r.insert, r.action, r.valLen, nullptr, nullptr, nullptr, r.predNum, r.predActor, r.predCtr};
  PcOut o; if (!field[cx]) return o;
  o.u = field[cx] + (cx == CX_PRED_ACTOR || cx == CX_PRED_CTR ? predBase : rowBase);
  if (cx == CX_VAL_LEN) { o.off = r.valOff + rowBase; o.base = valBase; o.sum = sum; }
  if (cx == CX_PRED_NUM) { o.off = r.predOff + rowBase; o.sum = sum; }
  return o;
}

// ---------------------------------------------------------------- the document chunk's columns (columnar.js:60-94)
// Op columns, one value per document row (the succ group: one per succ entry), in directory order.
enum DocColIx { OC_OBJ_ACTOR, OC_OBJ_CTR, OC_KEY_ACTOR, OC_KEY_CTR, OC_KEY_STR, OC_ID_ACTOR, OC_ID_CTR, OC_INSERT, OC_ACTION, OC_VAL_LEN,
                OC_VAL_RAW, OC_CHLD_ACTOR, OC_CHLD_CTR, OC_SUCC_NUM, OC_SUCC_ACTOR, OC_SUCC_CTR, NUM_DOC_COLS };
static const u32 DOC_COL_IDS[NUM_DOC_COLS] = {0x01, 0x02, 0x11, 0x13, 0x15, 0x21, 0x23, 0x34, 0x42, 0x56, 0x57, 0x61, 0x63, 0x80, 0x81, 0x83};
static const u32 ALL_DOC_COLS = (1u << NUM_DOC_COLS) - 1;
static const u32 DECODED_DOC_COLS = ALL_DOC_COLS & ~((1u << OC_VAL_RAW) | (1u << OC_CHLD_ACTOR) | (1u << OC_CHLD_CTR));   // valRaw is read through valLen; child columns are always empty
struct DocCols { u32 off[NUM_DOC_COLS]; u32 len[NUM_DOC_COLS]; };   // arena ranges (len 0: absent)
// The change column decoder that reads op column k (-1: none). idActor / idCtr have no change column of their own: they
// are read as objActor (RLE uint) and keyCtr (delta) into the rows doc_col_rows() puts in those fields' place.
HD int doc_col_decoder(int k) {   // (the succ group has the pred group's layout)
  const signed char cx[NUM_DOC_COLS] = {CX_OBJ_ACTOR, CX_OBJ_CTR, CX_KEY_ACTOR, CX_KEY_CTR, CX_KEY_STR, CX_OBJ_ACTOR, CX_KEY_CTR, CX_INSERT, CX_ACTION,
                                        CX_VAL_LEN, -1, -1, -1, CX_PRED_NUM, CX_PRED_ACTOR, CX_PRED_CTR};
  return cx[k];
}
HD RawRows doc_col_rows(int k, RawRows r, u32* idActor, u32* idCtr) { if (k == OC_ID_ACTOR) r.objActor = idActor; if (k == OC_ID_CTR) r.keyCtr = idCtr; return r; }

// Change metadata columns, one value per change (depsIndex: one per dependency). lc: LoadedColKernel's reader, pk: the parallel decoder.
enum ChangeColIx { CC_ACTOR, CC_SEQ, CC_MAX_OP, CC_TIME, CC_MESSAGE, CC_DEPS_NUM, CC_DEPS_INDEX, CC_EXTRA_LEN, CC_EXTRA_RAW, NUM_CHANGE_COLS };
struct ChangeColDef { u32 id; int lc, pk; };
static const ChangeColDef CHANGE_COLS[NUM_CHANGE_COLS] = {
  {0x01, LC_UINT, PK_UINT}, {0x03, LC_DELTA, PK_DELTA}, {0x13, LC_DELTA, PK_DELTA}, {0x23, LC_DELTA, PK_DELTA}, {0x35, LC_STRING, PK_NONE},
  {0x40, LC_UINT, PK_UINT}, {0x43, LC_DELTA, PK_DELTA}, {0x56, LC_EXTRA_LEN, PK_EXTRA_LEN}, {0x57, -1, PK_NONE}};

}  // namespace amg
