// amgpu — kernels #1: columnar change decode.
//
// Replaces (reference paths relative to /root/reference):
//   backend/columnar.js:688-708  decodeContainerHeader (magic, SHA-256 over [type|len|body], checksum)   -> ShaKernel / sha_change
//   backend/columnar.js:635-652  decodeChangeHeader, :609-624 decodeColumnInfo, :741-765 decodeChangeColumns -> parse_change
//   backend/encoding.js:341-488  LEB128 readers, :789-920 RLEDecoder, :1004-1051 DeltaDecoder,
//   backend/encoding.js:1141-1207 BooleanDecoder, backend/new.js:570-610 readOperation               -> fast_value / decode_one_column_t
//   backend/new.js:678-724       readNextChangeOp (opId assignment, reference validation)             -> FinalizeOpsKernel (gate.cuh)
//
// Layout: all change bytes of a call sit back to back in one device arena (u8). The apply path decodes with ONE fused kernel,
// k_decode_tiles (below: one CTA = 128 consecutive changes staged in shared memory by a bulk copy, one thread per change:
// header -> 48-byte ChangeHot + counts, columns -> raw u32 rows in structure-of-arrays form, row ranges from a global cursor);
// changes of more than SMALL_CHANGE_OPS ops only reserve rows there and are expanded by DecodeColumnKernel (one thread per
// (column, change)) or the parallel decoders of doccols.cuh. save() re-parses headers with ParseKernel (ChangeMeta: the fields
// only it needs). The finalize kernel packs raw rows into 64-bit ids with document-global actor numbers.
#pragma once
#include "common.cuh"

namespace amg {

static const u32 NULL32 = 0xffffffffu;
static const int NCOLS = 14;   // known change columns, in this order:
static const u32 SMALL_CHANGE_OPS = 16;   // changes with at most this many ops are decoded by one thread inside k_decode_tiles
enum ColIx { CX_OBJ_ACTOR = 0, CX_OBJ_CTR, CX_KEY_ACTOR, CX_KEY_CTR, CX_KEY_STR, CX_INSERT, CX_ACTION, CX_VAL_LEN, CX_VAL_RAW,
             CX_CHLD_ACTOR, CX_CHLD_CTR, CX_PRED_NUM, CX_PRED_ACTOR, CX_PRED_CTR };
// A column id this version does not know is carried along (unknowncols.hpp) - except a GROUP_CARD column (type 0) whose group
// (id >> 4) is one of the groups the known scalar columns live in (obj 0, key 1, insert 3, action 4, value 5, child 6): the
// reference's readOperation would then read those known columns as arrays (new.js:576-597). No encoder writes that; refused.
HD bool groups_known_columns(u32 columnId) { return (columnId & 7u) == 0 && (columnId >> 4) < 7u && (columnId >> 4) != 2u; }
HD int col_index_of(u32 columnId) {
  switch (columnId) {
    case 0x01: return CX_OBJ_ACTOR; case 0x02: return CX_OBJ_CTR; case 0x11: return CX_KEY_ACTOR; case 0x13: return CX_KEY_CTR;
    case 0x15: return CX_KEY_STR; case 0x34: return CX_INSERT; case 0x42: return CX_ACTION; case 0x56: return CX_VAL_LEN;
    case 0x57: return CX_VAL_RAW; case 0x61: return CX_CHLD_ACTOR; case 0x63: return CX_CHLD_CTR; case 0x70: return CX_PRED_NUM;
    case 0x71: return CX_PRED_ACTOR; case 0x73: return CX_PRED_CTR; default: return -1;
  }
}

// error codes raised by kernels (ordered by the reference's check order where it matters)
enum KErr {
  KE_NONE = 0, KE_MAGIC, KE_CHECKSUM, KE_TRAILING, KE_CHUNK_TYPE, KE_TRUNCATED, KE_NUM_RANGE, KE_COL_ORDER, KE_COL_DEFLATE,
  KE_RLE_REP1, KE_RLE_SUCC_REP, KE_RLE_SUCC_LIT, KE_RLE_SUCC_NULL, KE_RLE_ZERO_NULL, KE_RLE_LIT_REP, KE_BOOL_ZERO,
  KE_OBJ_MISMATCH, KE_KEY_MISMATCH, KE_ACTOR_INDEX, KE_TOO_LARGE, KE_UNKNOWN_ACTOR, KE_PRED_MISSING, KE_REF_ELEM, KE_DUP_OPID,
  KE_UNSUPPORTED_OP, KE_LAMPORT, KE_HASH_COLLISION, KE_LIST_ELEM, KE_PRED_ORDER, KE_DEFLATE, KE_UNKNOWN_COUNTER, KE_HIST_RANGE, KE_HIST_OPID, KE_HIST_DEP, KE_FLOAT_LEN /* columnar.js:316 */,
  KE_SUBARRAY,  // raw bytes (a string, a hash, a column, a chunk body) reach past the end: encoding.js:497, where a number that runs out is KE_TRUNCATED (:353)
  KE_GROUP_COLUMN   // an unknown GROUP_CARD column in the group of known scalar columns: readOperation (new.js:576-597) would read those as arrays
};
// error word: (code << 32 | item index); the smallest item index wins so that the error reported is
// the one the sequential reference would hit first within a phase.
HD void raise(u64* errWord, u32 code, u64 item) {
  u64 w = ((u64)(item & 0xffffffffu) << 8) | code;   // ordered by item, then code
#ifdef AMG_EMU
  if (*errWord == 0 || w < *errWord) *errWord = w;
#else
#ifdef __CUDA_ARCH__
  unsigned long long old = *errWord;
  while (old == 0 || w < old) { unsigned long long prev = atomicCAS(errWord, old, w); if (prev == old) break; old = prev; }
#endif
#endif
}

struct ChangeMeta {
  u32 off, len;            // absolute arena offset / length of the (inflated) change
  u32 depsOff, nDeps;      // first dependency hash (32 bytes each)
  u32 actorOff, actorLen;  // author actor id bytes
  u32 msgOff, msgLen;
  u32 otherOff, nOther;    // other-actor table entries (len-prefixed), after the count
  u32 extraOff, extraLen;  // trailing bytes
  u32 nOps, nPreds;
  u32 dirOff, dataOff;     // column directory entries / first column's data
  u64 seq, startOp; long long time;
};

// ---------------------------------------------------------------- byte-level readers
// Where the bytes come from: a plain pointer (global memory, host memory in the emulation build) or a CTA's shared-memory
// copy of its byte range (decode tile kernel). `pos` is always an absolute arena offset.
struct PtrSrc { const u8* base; HD u32 ld(u32 pos) const { return base[pos]; } };
#ifndef AMG_EMU
// sbase = 32-bit shared-memory address that holds arena byte 0 of this view (stage address - first staged arena offset); an
// explicit ld.shared: through a pointer the compiler lost the address space in most of the parser and emitted generic loads
// (L1TEX path, long scoreboard) for what is a shared-memory read
#ifndef AMG_DT_THREADS
#define AMG_DT_THREADS 128
#endif
struct SmemSrc {
  u32 sbase; u32 lutBase /* shared address of the 128-byte column-id -> column-index table */; u32 slotBase /* shared address of this thread's first value slot */;
  DEV u32 ld(u32 pos) const { u32 v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(sbase + pos)); return v; }
};
#endif

template <class S> struct ByteReaderT {
  S src; u32 pos, end; u32 err;
  HD ByteReaderT(S s, u32 p, u32 e) : src(s), pos(p), end(e), err(0) {}
  HD bool done() const { return pos >= end; }
  // encoding.js:416-441 readUint64 + :389-395 53-bit range check
  HD u64 uleb() {
    if (pos + 3 < end) {   // values of up to four bytes (28 bits: nearly all of them) in 32-bit arithmetic, without the 64-bit loop
      const u32 b0 = src.ld(pos);
      if (!(b0 & 0x80)) { pos++; return b0; }
      const u32 b1 = src.ld(pos + 1); u32 v = (b0 & 0x7f) | ((b1 & 0x7f) << 7);
      if (!(b1 & 0x80)) { pos += 2; return v; }
      const u32 b2 = src.ld(pos + 2); v |= (b2 & 0x7f) << 14;
      if (!(b2 & 0x80)) { pos += 3; return v; }
      const u32 b3 = src.ld(pos + 3); v |= (b3 & 0x7f) << 21;
      if (!(b3 & 0x80)) { pos += 4; return v; }
    }
    u64 result = 0; int shift = 0;
    while (pos < end) {
      const u32 b = src.ld(pos);
      if (shift == 63 && (b & 0xfe)) { err = KE_NUM_RANGE; return 0; }
      result |= (u64)(b & 0x7f) << shift; shift += 7; pos++;
      if (!(b & 0x80)) { if (result > ((1ULL << 53) - 1)) err = KE_NUM_RANGE; return result; }
    }
    err = KE_TRUNCATED; return 0;
  }
  // encoding.js:450-488 readInt64 + :402-408
  HD long long sleb() {
    if (pos + 1 < end) {
      const u32 b0 = src.ld(pos);
      if (!(b0 & 0x80)) { pos++; return (long long)((int)(b0 << 25) >> 25); }
      const u32 b1 = src.ld(pos + 1);
      if (!(b1 & 0x80)) { pos += 2; return (long long)((int)(((b0 & 0x7f) | (b1 << 7)) << 18) >> 18); }
    }
    u64 result = 0; int shift = 0;
    while (pos < end) {
      const u32 b = src.ld(pos);
      if (shift == 63 && b != 0 && b != 0x7f) { err = KE_NUM_RANGE; return 0; }
      result |= (u64)(b & 0x7f) << shift; shift += 7; pos++;
      if (!(b & 0x80)) {
        if ((b & 0x40) && shift < 64) result |= ~0ULL << shift;
        long long v = (long long)result;
        if (v < -((1LL << 53) - 1) || v > ((1LL << 53) - 1)) err = KE_NUM_RANGE;
        return v;
      }
    }
    err = KE_TRUNCATED; return 0;
  }
  HD void skip(u64 n) { if ((u64)pos + n > end) { err = KE_SUBARRAY; pos = end; } else pos += (u32)n; }   // readRawBytes: encoding.js:494-500
  // the same number, clamped to 32 bits: for lengths and counts, where anything that large is an error a few lines later
  HD u32 ulebc() {
    if (pos + 3 < end) {
      const u32 b0 = src.ld(pos);
      if (!(b0 & 0x80)) { pos++; return b0; }
      const u32 b1 = src.ld(pos + 1); u32 v = (b0 & 0x7f) | ((b1 & 0x7f) << 7);
      if (!(b1 & 0x80)) { pos += 2; return v; }
    }
    const u64 v = uleb(); return v > 0xffffffffULL ? 0xffffffffu : (u32)v;
  }
  HD void skip32(u32 n) { if (pos > end || n > end - pos) { err = KE_SUBARRAY; pos = end; } else pos += n; }
};
struct ByteReader : ByteReaderT<PtrSrc> {
  const u8* base;
  HD ByteReader(const u8* b, u32 p, u32 e) : ByteReaderT<PtrSrc>(PtrSrc{b}, p, e), base(b) {}
};

// RLE record walker (encoding.js:789-920) over numeric (uint / int) or utf8 columns. One value at a time.
template <class S> struct RleReaderT {
  ByteReaderT<S> r; int type;   // 0 uint, 1 int, 2 utf8
  long long count; int state;   // 0 none, 1 repetition, 2 literal, 3 nulls
  long long lastNum; u32 lastOff, lastLen; bool haveLast; bool lastNull;
  HD RleReaderT(S s, u32 p, u32 e, int t) : r(s, p, e), type(t), count(0), state(0), lastNum(0), lastOff(0), lastLen(0), haveLast(false), lastNull(false) {}
  HD bool done() const { return count == 0 && r.done(); }
  HD bool strEq(u32 offA, u32 lenA, u32 offB, u32 lenB) const {
    if (lenA != lenB) return false;
    for (u32 i = 0; i < lenA; i++) if (r.src.ld(offA + i) != r.src.ld(offB + i)) return false;
    return true;
  }
  HD void readRaw(long long& num, u32& off, u32& len) {
    if (type == 0) num = (long long)r.uleb();
    else if (type == 1) num = r.sleb();
    else { u64 l = r.uleb(); off = r.pos; len = (u32)l; r.skip(l); }
  }
  HD bool sameAsLast(long long num, u32 off, u32 len) const {
    if (!haveLast || lastNull) return false;
    return type == 2 ? strEq(off, len, lastOff, lastLen) : num == lastNum;
  }
  // returns false for null; value in num (numeric) or off/len (utf8)
  HD bool next(long long& num, u32& off, u32& len) {
    if (done()) return false;
    if (count == 0) {   // readRecord
      count = r.sleb();
      if (r.err) return false;
      if (count > 1) {
        long long n = 0; u32 o = 0, l = 0; readRaw(n, o, l);
        if ((state == 1 || state == 2) && sameAsLast(n, o, l)) r.err = KE_RLE_SUCC_REP;
        state = 1; lastNum = n; lastOff = o; lastLen = l; haveLast = true; lastNull = false;
      } else if (count == 1) { r.err = KE_RLE_REP1; return false; }
      else if (count < 0) { count = -count; if (state == 2) r.err = KE_RLE_SUCC_LIT; state = 2; }
      else {
        if (state == 3) r.err = KE_RLE_SUCC_NULL;
        count = (long long)r.uleb();
        if (count == 0) { r.err = KE_RLE_ZERO_NULL; return false; }
        state = 3; haveLast = true; lastNull = true;
      }
    }
    count -= 1;
    if (state == 2) {
      long long n = 0; u32 o = 0, l = 0; readRaw(n, o, l);
      if (sameAsLast(n, o, l)) r.err = KE_RLE_LIT_REP;
      lastNum = n; lastOff = o; lastLen = l; haveLast = true; lastNull = false;
      num = n; off = o; len = l; return true;
    }
    if (state == 3) return false;
    num = lastNum; off = lastOff; len = lastLen; return true;
  }
};
struct RleReader : RleReaderT<PtrSrc> { HD RleReader(const u8* b, u32 p, u32 e, int t) : RleReaderT<PtrSrc>(PtrSrc{b}, p, e, t) {} };

// ---------------------------------------------------------------- SHA-256 (FIPS 180-4), one thread per change
struct ShaConsts { u32 k[64]; };
#ifndef AMG_EMU
__constant__ ShaConsts c_sha;
#endif
static const u32 SHA_K[64] = {
  0x428a2f98,0x71374491,0xb5c0fbcf,0xe9b5dba5,0x3956c25b,0x59f111f1,0x923f82a4,0xab1c5ed5,0xd807aa98,0x12835b01,0x243185be,0x550c7dc3,
  0x72be5d74,0x80deb1fe,0x9bdc06a7,0xc19bf174,0xe49b69c1,0xefbe4786,0x0fc19dc6,0x240ca1cc,0x2de92c6f,0x4a7484aa,0x5cb0a9dc,0x76f988da,
  0x983e5152,0xa831c66d,0xb00327c8,0xbf597fc7,0xc6e00bf3,0xd5a79147,0x06ca6351,0x14292967,0x27b70a85,0x2e1b2138,0x4d2c6dfc,0x53380d13,
  0x650a7354,0x766a0abb,0x81c2c92e,0x92722c85,0xa2bfe8a1,0xa81a664b,0xc24b8b70,0xc76c51a3,0xd192e819,0xd6990624,0xf40e3585,0x106aa070,
  0x19a4c116,0x1e376c08,0x2748774c,0x34b0bcb5,0x391c0cb3,0x4ed8aa4a,0x5b9cca4f,0x682e6ff3,0x748f82ee,0x78a5636f,0x84c87814,0x8cc70208,
  0x90befffa,0xa4506ceb,0xbef9a3f7,0xc67178f2};

HD u32 rotr32(u32 x, int n) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(x, x, n);
#else
  return (x >> n) | (x << (32 - n));
#endif
}
// rotr(x,a) ^ rotr(x,b) ^ (SHIFT ? x >> c : rotr(x,c)): three funnel shifts and one LOP3. (Measured and dropped: the rotations
// as halves of 64-bit products on the FMA pipe - IMAD.WIDE with multipliers from constant memory - to relieve the ALU pipe:
// 0.59 ms instead of 0.42 ms for the 1M changes of C3.)
template <int A, int B, int C, bool SHIFT> HD u32 sha_sigma(u32 x) { return rotr32(x, A) ^ rotr32(x, B) ^ (SHIFT ? (x >> C) : rotr32(x, C)); }
// big-endian 32-bit load at an arbitrary byte address (two aligned loads + funnel shift on device)
HD u32 load_be32(const u8* p) {
#if defined(__CUDA_ARCH__)
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const u32* w = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
  const u32 sh = (u32)(a & 3) * 8;
  const u32 lo = w[0], hi = sh ? w[1] : 0;
  return __byte_perm(__funnelshift_r(lo, hi, sh), 0, 0x0123);
#else
  return (u32)p[0] << 24 | (u32)p[1] << 16 | (u32)p[2] << 8 | p[3];
#endif
}
// One compression: 16 rounds on the message words as they are, then 3 x 16 rounds with the message schedule. Inside a
// 16-round body every w[] index is a compile-time constant (the schedule stays in registers) while the code stays small
// enough for the instruction cache (a fully unrolled 64-round body made ShaKernel stall on instruction fetch: ncu
// "no_instruction"); the first 16 rounds are peeled so that no round carries a "schedule or not" test.
template <bool SCHEDULE> HD void sha256_rounds16(u32& a, u32& b, u32& c, u32& d, u32& e, u32& f, u32& g, u32& hh, u32* w, const u32* K) {
#pragma unroll
  for (int j = 0; j < 16; j++) {
    if (SCHEDULE) {
      const u32 w15 = w[(j + 1) & 15], w2 = w[(j + 14) & 15];
      const u32 s0 = sha_sigma<7, 18, 3, true>(w15), s1 = sha_sigma<17, 19, 10, true>(w2);
      w[j] = w[j] + s0 + w[(j + 9) & 15] + s1;
    }
    const u32 t1 = hh + sha_sigma<6, 11, 25, false>(e) + ((e & f) ^ (~e & g)) + K[j] + w[j];
    const u32 t2 = sha_sigma<2, 13, 22, false>(a) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
}
HD void sha256_compress(u32* h, u32* w, const u32* K) {
  u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  sha256_rounds16<false>(a, b, c, d, e, f, g, hh, w, K);
#pragma unroll 1
  for (int r = 16; r < 64; r += 16) sha256_rounds16<true>(a, b, c, d, e, f, g, hh, w, K + r);
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// Where the bytes of ONE change are read from when it is hashed: global (host, in the emulation) memory. byte(i) = byte i of the change; on the device word(k) = aligned 32-bit word k counted from
// the aligned word that holds the first message byte (the message = bytes 8 ..), mis() = the message's misalignment.
struct GlobalBytes {
  const u8* p;
  HD u32 byte(u32 i) const { return p[i]; }
#if defined(__CUDA_ARCH__)
  DEV u32 mis() const { return (u32)(reinterpret_cast<uintptr_t>(p + 8) & 3); }
  DEV u32 word(u32 k) const { return reinterpret_cast<const u32*>(p + 8 - mis())[k]; }   // (pointer arithmetic on p: the loads stay global loads)
#endif
};
// SHA-256 of bytes 8 .. len of change c (columnar.js:688-708: the hash covers everything behind the checksum); writes the
// 32-byte digest, checks magic and checksum. DEFLATEd changes (chunk type 2, columnar.js:742) are left out when the caller
// hashes them later, once they are inflated.
template <class BS> HD void sha_change(const BS& bs, size_t c, u32 len, u8* hashOut, u64* errWord, bool deflatedLater) {
  if (len > 8 && bs.byte(8) == 2 && bs.byte(0) == 0x85) {
    if (!deflatedLater) raise(errWord, KE_CHUNK_TYPE, c);
    return;
  }
  if (len < 10 || bs.byte(0) != 0x85 || bs.byte(1) != 0x6f || bs.byte(2) != 0x4a || bs.byte(3) != 0x83) { raise(errWord, KE_MAGIC, c); return; }
#if defined(__CUDA_ARCH__)
  const u32* K = c_sha.k;
#else
  const u32* K = SHA_K;
#endif
  u32 h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  const u32 mlen = len - 8;
  // blocks: all full 64-byte blocks, then one or two padded blocks (0x80, zeros, 64-bit bit length). Message word i of a
  // block = 4 bytes at an arbitrary address: two aligned 32-bit loads (the second is the next word's first), funnel shift,
  // byte swap. Full blocks take the words as they are; in the padded blocks every word is masked by how many message bytes
  // it still holds (branch-free), and no load reaches more than one word past the message.
  const u32 nBlocks = (mlen + 9 + 63) / 64; u32 w[16];
#if defined(__CUDA_ARCH__)
  const u32 sh = bs.mis() * 8, lastAligned = (mlen + bs.mis() + 3) / 4;   // aligned words [0, lastAligned) hold message bytes
#endif
  for (u32 blk = 0; blk < nBlocks; blk++) {
    const u32 done = blk * 64;
#if defined(__CUDA_ARCH__)
    const u32 k0 = done / 4;
    if (done + 64 <= mlen) {
      u32 lo = bs.word(k0);
#pragma unroll
      for (int i = 0; i < 16; i++) { const u32 hi = bs.word(k0 + i + 1); w[i] = __byte_perm(__funnelshift_r(lo, hi, sh), 0, 0x0123); lo = hi; }
    } else {
      u32 lo = bs.word(k0 < lastAligned ? k0 : lastAligned);
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const u32 k = k0 + i + 1, hi = bs.word(k < lastAligned ? k : lastAligned);
        const u32 v = __byte_perm(__funnelshift_r(lo, hi, sh), 0, 0x0123);
        const int rem = (int)mlen - (int)(done + 4 * i);   // message bytes from this word on
        const u32 r8 = 8u * (u32)(rem < 0 ? 0 : (rem > 4 ? 4 : rem));
        const u32 keep = ~__funnelshift_rc(0xffffffffu, 0u, r8), pad = rem < 0 ? 0u : __funnelshift_rc(0x80000000u, 0u, r8);
        w[i] = (v & keep) | pad; lo = hi;
      }
    }
#else
    for (int i = 0; i < 16; i++) {
      u32 v = 0;
      for (int b = 0; b < 4; b++) { const u32 ix = done + 4 * i + b; u32 byte = 0; if (ix < mlen) byte = bs.byte(8 + ix); else if (ix == mlen) byte = 0x80; v = (v << 8) | byte; }
      w[i] = v;
    }
#endif
    if (blk == nBlocks - 1) { w[14] = (u32)(((u64)mlen * 8) >> 32); w[15] = (u32)((u64)mlen * 8); }
    sha256_compress(h, w, K);
  }
  u8* out = hashOut + c * 32;
#if defined(__CUDA_ARCH__)
  uint4* o4 = reinterpret_cast<uint4*>(out);   // digests are 32-byte aligned
  o4[0] = make_uint4(__byte_perm(h[0], 0, 0x0123), __byte_perm(h[1], 0, 0x0123), __byte_perm(h[2], 0, 0x0123), __byte_perm(h[3], 0, 0x0123));
  o4[1] = make_uint4(__byte_perm(h[4], 0, 0x0123), __byte_perm(h[5], 0, 0x0123), __byte_perm(h[6], 0, 0x0123), __byte_perm(h[7], 0, 0x0123));
#else
  for (int i = 0; i < 8; i++) { out[4 * i] = h[i] >> 24; out[4 * i + 1] = h[i] >> 16; out[4 * i + 2] = h[i] >> 8; out[4 * i + 3] = h[i]; }
#endif
  if (h[0] != ((bs.byte(4) << 24) | (bs.byte(5) << 16) | (bs.byte(6) << 8) | bs.byte(7))) raise(errWord, KE_CHECKSUM, c);
}
// one change per thread, bytes read where they lie
struct ShaKernel {
  const u8* arena; const u32* chOff; const u32* chLen; u8* hashOut /* [n][32] */; u64* errWord; const u32* subset /* optional: only these changes */; u32* deflList /* non-null: DEFLATEd changes are skipped (hashed once inflated) */;
  size_t first = 0;   // items are changes first, first + 1, ...
  HD void operator()(size_t ci) const {
    const size_t c = subset ? subset[ci] : first + ci;
    sha_change(GlobalBytes{arena + chOff[c]}, c, chLen[c], hashOut, errWord, deflList != nullptr);
  }
};

#ifndef AMG_SHA_MINBLOCKS
#define AMG_SHA_MINBLOCKS 3
#endif
template <> struct LaunchTraits<ShaKernel> { static const int minBlocks = AMG_SHA_MINBLOCKS; };
// ---- SHA-256 of the changes first .. end-1 of a batch: one thread per change, bytes read where they lie (ShaKernel). (Measured
// and dropped: staging a tile's bytes in shared memory like the decode does - 0.52 ms instead of 0.42 ms on C3: the kernel is
// bound by the rounds on the ALU pipe, not by its loads.)
struct ShaTilesArgs { const u8* arena; const u32* chOff; const u32* chLen; u8* hashOut; u64* errWord; u32* deflList /* non-null: DEFLATEd changes are hashed later */; u32 first, end; };
inline void sha_range(Ctx& c, const ShaTilesArgs& a, bool onSide) {
  if (a.end <= a.first) return;
  ShaKernel sk{a.arena, a.chOff, a.chLen, a.hashOut, a.errWord, nullptr, a.deflList}; sk.first = a.first;
  foreach(c, a.end - a.first, sk, onSide);
}

// number of values in an RLE column (record-level: runs are not expanded); *err receives a KErr
template <class S> HD u32 rle_count_values_t(const S& src, u32 off, u32 end, u32* err, int type = 0 /* 0 uint, 1 int, 2 utf8 */) {
  RleReaderT<S> a(src, off, end, type); u64 n = 0;
  while (!a.done() && !a.r.err) {
    long long v; u32 o, l; a.next(v, o, l);
    u64 adv = 1;
    if (a.state != 2 && a.count > 0) { adv += (u64)a.count; a.count = 0; }
    n += adv;
  }
  *err = a.r.err; if (n > 0xfffffffeULL) { *err = KE_TOO_LARGE; n = 0; }
  return (u32)n;
}
// sum of the first `limit` values of an RLE uint column (nulls count as 0)
template <class S> HD u64 rle_sum_values_t(const S& src, u32 off, u32 end, u32 limit, u32* err) {
  RleReaderT<S> pn(src, off, end, 0); u32 seen = 0; u64 sum = 0;
  while (!pn.done() && !pn.r.err && seen < limit) {
    long long n = 0; u32 o, l; const bool nn = pn.next(n, o, l);
    u64 adv = 1;
    if (pn.state != 2 && pn.count > 0) { adv += (u64)pn.count; if (seen + adv > limit) adv = limit - seen; pn.count -= (long long)(adv - 1); }
    if (nn) sum += (u64)n * adv;
    seen += (u32)adv;
  }
  *err = pn.r.err; return sum;
}
HD u32 rle_count_values(const u8* arena, u32 off, u32 end, u32* err) { return rle_count_values_t(PtrSrc{arena}, off, end, err); }
// decodeValue (columnar.js:300-329) of the payload arena[valOff, valOff + (valLen >> 4)): numbers must be complete LEB128
// values within 53 bits, floating point payloads must be 8 bytes. Returns a KErr (0 = the value decodes).
HD u32 decode_value_error(const u8* arena, u32 valLen, u32 valOff) {
  const u32 tag = valLen & 15, n = valLen >> 4;
  if (tag == 3 || tag == 4 || tag == 8 || tag == 9) {
    ByteReader r(arena, valOff, valOff + n);
    if (tag == 3) r.uleb(); else r.sleb();
    return r.err;
  }
  return tag == 5 && n != 8 ? (u32)KE_FLOAT_LEN : 0u;
}
HD u64 rle_sum_values(const u8* arena, u32 off, u32 end, u32 limit, u32* err) { return rle_sum_values_t(PtrSrc{arena}, off, end, limit, err); }

// ---------------------------------------------------------------- header / column directory parse, one thread per change
struct ParseKernel {
  const u8* arena; const u32* chOff; const u32* chLen; size_t numChanges;
  ChangeMeta* meta; u32* colOff /* [NCOLS][numChanges] */; u32* colLen; u32* nOpsOut; u32* nPredsOut; u32* nDepsOut; u32* nActorsOut; u64* errWord;
  u32* anyLarge /* set when some change has more than SMALL_CHANGE_OPS ops (else the large-change path is skipped entirely) */;
  HD void operator()(size_t c) const { (*this)(c, this->arena); }
  HD void operator()(size_t c, const u8* arena) const {   // `arena` may be the block's shared-memory copy (foreach_staged)
    const u32 off = chOff[c], len = chLen[c];
    ChangeMeta m; memset(&m, 0, sizeof(m)); m.off = off; m.len = len;
    nOpsOut[c] = 0; nPredsOut[c] = 0; nDepsOut[c] = 0; nActorsOut[c] = 1;
    ByteReader r(arena, off + 8, off + len);
    const u32 chunkType = r.done() ? 0xff : arena[r.pos]; r.pos++;
    const u64 chunkLen = r.uleb();
    if (r.err) { raise(errWord, r.err, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    if ((u64)r.pos + chunkLen > (u64)off + len) { raise(errWord, KE_TRUNCATED, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    if ((u64)r.pos + chunkLen != (u64)off + len) { raise(errWord, KE_TRAILING, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    if (chunkType != 1) { raise(errWord, KE_CHUNK_TYPE, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    // decodeChangeHeader
    const u64 nDeps = r.uleb(); m.depsOff = r.pos; m.nDeps = (u32)nDeps; r.skip(nDeps * 32);
    const u64 actorLen = r.uleb(); m.actorOff = r.pos; m.actorLen = (u32)actorLen; r.skip(actorLen);
    m.seq = r.uleb(); m.startOp = r.uleb(); m.time = r.sleb();
    const u64 msgLen = r.uleb(); m.msgOff = r.pos; m.msgLen = (u32)msgLen; r.skip(msgLen);
    const u64 nOther = r.uleb(); m.otherOff = r.pos; m.nOther = (u32)nOther;
    for (u64 i = 0; i < nOther && !r.err; i++) { u64 l = r.uleb(); r.skip(l); }
    // decodeColumnInfo
    const u64 nCols = r.uleb();
    if (r.err) { raise(errWord, r.err, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    const u32 dirPos = r.pos; long long lastId = -1; u64 total = 0;
    u32 actOff = 0, actLen = 0, pnOff = 0, pnLen = 0;   // the two columns needed for counting, relative to the data start
    for (u64 i = 0; i < nCols && !r.err; i++) {
      const u64 id = r.uleb(), l = r.uleb();
      if (lastId >= 0 && ((u32)id & ~8u) <= ((u32)lastId & ~8u)) { raise(errWord, KE_COL_ORDER, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
      if (id & 8) { raise(errWord, KE_COL_DEFLATE, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
      if (id == 0x42) { actOff = (u32)total; actLen = (u32)l; } else if (id == 0x70) { pnOff = (u32)total; pnLen = (u32)l; }
      lastId = (long long)id; total += l;
    }
    if (r.err) { raise(errWord, r.err, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    const u32 dataPos = r.pos;
    if ((u64)dataPos + total > (u64)off + len) { raise(errWord, KE_TRUNCATED, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    m.dirOff = dirPos; m.dataOff = dataPos;
    m.extraOff = dataPos + (u32)total; m.extraLen = off + len - m.extraOff;
    // count ops (values of the action column) and preds (sum of the predNum column)
    u32 kerr = 0; u32 nOps; u64 nPreds = 0;
    // single-op changes (the shape of editing traces): both columns are one literal record [-1, value]
    const u8* ap = arena + dataPos + actOff; const u8* pp = arena + dataPos + pnOff;
    if (actLen == 2 && ap[0] == 0x7f && ap[1] < 0x80 && ((pnLen == 2 && pp[0] == 0x7f && pp[1] < 0x80) || pnLen == 0)) { nOps = 1; nPreds = pnLen ? pp[1] : 0; }
    else {
      nOps = rle_count_values(arena, dataPos + actOff, dataPos + actOff + actLen, &kerr);
      if (!kerr) nPreds = rle_sum_values(arena, dataPos + pnOff, dataPos + pnOff + pnLen, nOps, &kerr);
    }
    if (kerr) { raise(errWord, kerr, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    if (nPreds > 0x7fffffffULL) { raise(errWord, KE_TOO_LARGE, c); m.nDeps = 0; m.nOther = 0; m.nOps = 0; m.nPreds = 0; meta[c] = m; return; }
    m.nOps = nOps; m.nPreds = (u32)nPreds;
    if (nOps > SMALL_CHANGE_OPS) {   // large change: publish the directory for the (column, change)-parallel kernel
      *anyLarge = 1;
      ByteReader d(arena, dirPos, dataPos); u32 pos = dataPos;
      for (int k = 0; k < NCOLS; k++) { colOff[(size_t)k * numChanges + c] = 0; colLen[(size_t)k * numChanges + c] = 0; }
      for (u64 i = 0; i < nCols; i++) {
        const u64 id = d.uleb(), l = d.uleb(); const int ix = col_index_of((u32)id);
        if (ix >= 0) { colOff[(size_t)ix * numChanges + c] = pos; colLen[(size_t)ix * numChanges + c] = (u32)l; }
        pos += (u32)l;
      }
    }
    meta[c] = m; nOpsOut[c] = nOps; nPredsOut[c] = (u32)nPreds; nDepsOut[c] = m.nDeps; nActorsOut[c] = 1 + m.nOther;
  }
};

// ---------------------------------------------------------------- column expansion
struct RawRows {   // SoA, one entry per op of the batch (raw change-local values; NULL32 = null)
  u32 *objActor, *objCtr, *keyActor, *keyCtr, *keyStrOff, *keyStrLen, *insert, *action, *valLen, *valOff, *predNum, *predOff;
  u32 *predActor, *predCtr;   // one entry per pred of the batch
};

// Expands one column of one change into the raw rows. Returns a KErr code (0 = ok).
template <class S> HD u32 decode_one_column_t(const S& arena, int col, u32 nOps, u32 base, u32 cOff, u32 cEnd, u32 valRawOff, u32 valRawLen, u32 predBase, u32 nPreds, const RawRows& rows) {
  u32 kerr = 0;
  switch (col) {
    case CX_OBJ_ACTOR: case CX_OBJ_CTR: case CX_KEY_ACTOR: case CX_ACTION: case CX_VAL_LEN: case CX_PRED_NUM: {
      u32* out = col == CX_OBJ_ACTOR ? rows.objActor : col == CX_OBJ_CTR ? rows.objCtr : col == CX_KEY_ACTOR ? rows.keyActor
               : col == CX_ACTION ? rows.action : col == CX_VAL_LEN ? rows.valLen : rows.predNum;
      RleReaderT<S> r(arena, cOff, cEnd, 0);
      u32 running = 0;   // VAL_LEN: byte offset into valRaw; PRED_NUM: pred offset
      const u32 rawBase = col == CX_VAL_LEN ? valRawOff : (col == CX_PRED_NUM ? predBase : 0);
      for (u32 i = 0; i < nOps; i++) {
        long long n = 0; u32 o, l; const bool nn = r.next(n, o, l);
        if (nn && (u64)n > 0xfffffffeULL) kerr = KE_TOO_LARGE;
        out[base + i] = nn ? (u32)n : NULL32;
        if (col == CX_VAL_LEN) { rows.valOff[base + i] = rawBase + running; running += nn ? (u32)((u64)n >> 4) : 0; }
        if (col == CX_PRED_NUM) { rows.predOff[base + i] = rawBase + running; running += nn ? (u32)n : 0; if (!nn) out[base + i] = 0; }
      }
      if (col == CX_VAL_LEN && running > valRawLen) kerr = KE_SUBARRAY;
      if (!kerr) kerr = r.r.err;
      break;
    }
    case CX_KEY_CTR: {
      RleReaderT<S> r(arena, cOff, cEnd, 1); long long acc = 0;
      for (u32 i = 0; i < nOps; i++) {
        long long n = 0; u32 o, l; const bool nn = r.next(n, o, l);
        if (nn) { acc += n; if (acc < 0 || acc > 0xfffffffeLL) kerr = KE_TOO_LARGE; }
        rows.keyCtr[base + i] = nn ? (u32)acc : NULL32;
      }
      if (!kerr) kerr = r.r.err;
      break;
    }
    case CX_KEY_STR: {
      RleReaderT<S> r(arena, cOff, cEnd, 2);
      for (u32 i = 0; i < nOps; i++) {
        long long n; u32 o = 0, l = 0; const bool nn = r.next(n, o, l);
        rows.keyStrOff[base + i] = nn ? o : 0; rows.keyStrLen[base + i] = nn ? l : NULL32;
      }
      kerr = r.r.err;
      break;
    }
    case CX_INSERT: {   // BooleanDecoder encoding.js:1141-1207
      ByteReaderT<S> r(arena, cOff, cEnd); bool val = true, first = true; u64 count = 0;
      for (u32 i = 0; i < nOps; i++) {
        bool v = false;
        if (!(count == 0 && r.done())) {
          while (count == 0) {
            count = r.uleb(); val = !val;
            if (r.err) break;
            if (count == 0 && !first) { kerr = KE_BOOL_ZERO; break; }
            first = false;
          }
          if (r.err || kerr) break;
          count--; v = val;
        }
        rows.insert[base + i] = v ? 1u : 0u;
      }
      if (!kerr) kerr = r.err;
      break;
    }
    case CX_PRED_ACTOR: case CX_PRED_CTR: {
      RleReaderT<S> r(arena, cOff, cEnd, col == CX_PRED_CTR ? 1 : 0); long long acc = 0;
      for (u32 j = 0; j < nPreds; j++) {
        long long n = 0; u32 o, l; const bool nn = r.next(n, o, l);
        if (col == CX_PRED_CTR) { if (nn) { acc += n; if (acc < 0 || acc > 0xfffffffeLL) kerr = KE_TOO_LARGE; } rows.predCtr[predBase + j] = nn ? (u32)acc : NULL32; }
        else { if (nn && (u64)n > 0xfffffffeULL) kerr = KE_TOO_LARGE; rows.predActor[predBase + j] = nn ? (u32)n : NULL32; }
      }
      if (!kerr) kerr = r.r.err;
      break;
    }
    default: break;   // VAL_RAW is referenced in place; chld* columns are not needed by the op set
  }
  return kerr;
}
HD u32 decode_one_column(const u8* arena, int col, u32 nOps, u32 base, u32 cOff, u32 cEnd, u32 valRawOff, u32 valRawLen, u32 predBase, u32 nPreds, const RawRows& rows) {
  return decode_one_column_t(PtrSrc{arena}, col, nOps, base, cOff, cEnd, valRawOff, valRawLen, predBase, nPreds, rows);
}
// default (column absent) values of the rows of one change
HD void fill_absent_column(int col, u32 nOps, u32 base, u32 predBase, u32 nPreds, const RawRows& rows) {
  u32* out = nullptr; u32 v = NULL32;
  switch (col) {
    case CX_OBJ_ACTOR: out = rows.objActor; break; case CX_OBJ_CTR: out = rows.objCtr; break; case CX_KEY_ACTOR: out = rows.keyActor; break;
    case CX_KEY_CTR: out = rows.keyCtr; break; case CX_ACTION: out = rows.action; break; case CX_VAL_LEN: out = rows.valLen; break;
    case CX_KEY_STR: for (u32 i = 0; i < nOps; i++) { rows.keyStrOff[base + i] = 0; rows.keyStrLen[base + i] = NULL32; } return;
    case CX_INSERT: out = rows.insert; v = 0; break;
    case CX_PRED_NUM: for (u32 i = 0; i < nOps; i++) { rows.predNum[base + i] = 0; rows.predOff[base + i] = predBase; } return;
    case CX_PRED_ACTOR: for (u32 j = 0; j < nPreds; j++) rows.predActor[predBase + j] = NULL32; return;
    case CX_PRED_CTR: for (u32 j = 0; j < nPreds; j++) rows.predCtr[predBase + j] = NULL32; return;
    default: return;
  }
  for (u32 i = 0; i < nOps; i++) out[base + i] = v;
  if (col == CX_VAL_LEN) for (u32 i = 0; i < nOps; i++) rows.valOff[base + i] = 0;
}

// ---------------------------------------------------------------- fused decode: header parse + column expansion in one pass
// What the rest of the apply pipeline needs of a change header: 48 bytes, written with three 128-bit stores (the counts
// that feed prefix sums - ops, preds, deps, actors - are separate u32 arrays). time / message / extra bytes are only
// needed by save(), which parses the headers again (ParseKernel above).
struct alignas(16) ChangeHot {
  u32 off, len, depsOff, actorOff;         // absolute arena offsets
  u32 actorLen, otherOff, dirOff, dataOff; // otherOff: first other-actor entry; dirOff / dataOff: column directory / first column's bytes
  u64 startOp, seq;
};

// One column that holds exactly one value: either the literal record [-1, v] or the null run [0, 1] (boolean: one run).
// Returns false for anything else (the general decoder then handles - and validates - the column).
template <class S> HD bool single_value(const S& src, int ix, u32 pos, u32 l, u32& v, bool& isNull, u32& used) {
  const u32 p0 = l > 0 ? src.ld(pos) : 0xffu, p1 = l > 1 ? src.ld(pos + 1) : 0xffu;
  if (ix == CX_INSERT) {
    if (l == 1 && p0 == 1) { v = 0; isNull = false; used = 1; return true; }
    if (l == 2 && p0 == 0 && p1 == 1) { v = 1; isNull = false; used = 2; return true; }
    return false;
  }
  isNull = false; v = 0; used = 0;
  if (l == 2 && p0 == 0 && p1 == 1) { isNull = true; used = 2; return true; }
  if (l < 2 || p0 != 0x7f) return false;
  if (ix == CX_KEY_STR) { if (p1 >= 0x80) return false; v = p1; used = 2 + v; return used == l; }
  // the literal's value: a LEB128 number of 1 .. 5 bytes that ends exactly at the column's end (counters of a long
  // document need three and four bytes)
  if (l > 6) return false;
  u64 val = p1 & 0x7fu; u32 last = p1; u32 nb = 1;
  if (l > 2) {   // more than one value byte
#pragma unroll
    for (u32 k = 1; k < 5; k++) if ((last & 0x80u) && nb < l - 1) { last = src.ld(pos + 1 + k); val |= (u64)(last & 0x7fu) << (7 * k); nb = k + 1; }
  }
  if ((last & 0x80u) || nb != l - 1) return false;
  used = l;
  if (ix == CX_KEY_CTR || ix == CX_PRED_CTR) {   // signed (delta from 0): negative values go to the general decoder, which reports them
    if (last & 0x40u) return false;
  }
  if (val > 0xfffffffeULL) return false;
  v = (u32)val;
  return true;
}
// The same test with the column index known at compile time (second phase of the fast walk in parse_change): the two
// common shapes - one literal byte, one null - are decided from (length, first byte, second byte) alone. Reads one byte past
// a column of length 0 or 1; the caller's bytes have that much slack (shared-memory window, zeroed arena tail).
template <int IX, class S> HD bool fast_value(const S& src, u32 pos, u32 l, u32& v) {
  const u32 p0 = src.ld(pos), p1 = src.ld(pos + 1);
  if (IX == CX_INSERT) {
    if (l == 1 && p0 == 1) { v = 0; return true; }
    if (l == 2 && p0 == 0 && p1 == 1) { v = 1; return true; }
    return false;
  }
  if (l == 2) {
    if (p0 == 0x7f && p1 < 0x80) {
      if ((IX == CX_KEY_CTR || IX == CX_PRED_CTR) && (p1 & 0x40u)) return false;   // negative delta: the general decoder reports it
      if (IX == CX_KEY_STR && p1 != 0) return false;
      v = p1; return true;
    }
    if (p0 == 0 && p1 == 1) { v = NULL32; return true; }
    return false;
  }
  if (l < 2 || p0 != 0x7f) return false;
  if (IX == CX_KEY_STR) { if (p1 >= 0x80) return false; v = p1; return 2 + v == l; }
  // longer numbers (2 .. 5 bytes of LEB128 that end exactly at the column's end): only for the columns that hold counters
  // and lengths; an actor index or an action that long is left to the general walk
  if (!(IX == CX_OBJ_CTR || IX == CX_KEY_CTR || IX == CX_VAL_LEN || IX == CX_PRED_CTR) || l > 6) return false;
  u64 val = p1 & 0x7fu; u32 last = p1; u32 nb = 1;
#pragma unroll
  for (u32 k = 1; k < 5; k++) if ((last & 0x80u) && nb < l - 1) { last = src.ld(pos + 1 + k); val |= (u64)(last & 0x7fu) << (7 * k); nb = k + 1; }
  if ((last & 0x80u) || nb != l - 1) return false;
  if ((IX == CX_KEY_CTR || IX == CX_PRED_CTR) && (last & 0x40u)) return false;
  if (val > 0xfffffffeULL) return false;
  v = (u32)val; return true;
}
// Per-thread scratch for the column values of a single-op change while its directory is walked: indexed by column
// index with an index that is not known at compile time. In registers that costs a divergent switch per column; the tile
// kernel keeps the 14 slots of a thread in shared memory (slot k of thread t at [k][t]: conflict-free) and looks the
// column index up in a 128-byte shared table; elsewhere (direct kernel, emulation) a local array and the switch do.
template <class S> struct ColSlots;
template <> struct ColSlots<PtrSrc> {
  u32 v[16];
  HD ColSlots(const PtrSrc&) {}
  HD void put(int ix, u32 x) { v[ix] = x; }
  HD u32 get(int ix) const { return v[ix]; }
  HD int index(u32 id) const { return col_index_of(id); }
};
#ifndef AMG_EMU
template <> struct ColSlots<SmemSrc> {
  u32 lutBase, slotBase;
  DEV ColSlots(const SmemSrc& s) : lutBase(s.lutBase), slotBase(s.slotBase) {}
  DEV void put(int ix, u32 x) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(slotBase + (u32)ix * (4u * AMG_DT_THREADS)), "r"(x) : "memory"); }
  DEV u32 get(int ix) const { u32 x; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(slotBase + (u32)ix * (4u * AMG_DT_THREADS)) : "memory"); return x; }
  DEV int index(u32 id) const { int x; asm volatile("ld.shared.s8 %0, [%1];" : "=r"(x) : "r"(lutBase + (id & 127u))); return x; }   // callers pass id < 128
};
#endif

// Result of the first walk over a change: header fields, counts, and - when every column holds exactly one value - the row,
// which stays in the thread's ColSlots (slot ix valid iff bit ix of `seen`) until its row index is known.
struct ParsedChange {
  ChangeHot h; u32 nDeps, nOther, nOps, nPreds; u32 err;   // err: KErr of the header / directory / count (raised for every change of a batch)
  bool single; bool unknownCols /* a column id this version does not know: the host carries its values (unknowncols.hpp) */;
  u32 seen, keyStrPos, valOff;
};
// columnar.js:688-708 (container), :635-652 decodeChangeHeader, :609-624 decodeColumnInfo; op count = values of the action
// column, pred count = sum of the predNum column (new.js:686-700 reads ops until the action column is exhausted)
template <class S> HD void parse_change(const S& src, ColSlots<S>& slots, u32 off, u32 len, ParsedChange& o) {
  o.h.off = off; o.h.len = len; o.h.depsOff = o.h.actorOff = o.h.actorLen = o.h.otherOff = o.h.dirOff = o.h.dataOff = 0; o.h.startOp = 0; o.h.seq = 0;
  o.nDeps = 0; o.nOther = 0; o.nOps = 0; o.nPreds = 0; o.err = 0; o.single = false; o.unknownCols = false; o.seen = 0; o.keyStrPos = 0; o.valOff = 0;
  const u32 end = off + len;
  ByteReaderT<S> r(src, off + 8, end);
  const u32 chunkType = r.done() ? 0xffu : src.ld(r.pos); r.pos++;
  const u64 chunkLen = r.uleb();
  if (r.err) { o.err = r.err; return; }
  if ((u64)r.pos + chunkLen > (u64)end) { o.err = KE_SUBARRAY; return; }
  if ((u64)r.pos + chunkLen != (u64)end) { o.err = KE_TRAILING; return; }
  if (chunkType != 1) { o.err = KE_CHUNK_TYPE; return; }
  // lengths and counts in 32-bit arithmetic (clamped: anything that does not fit is longer than the change)
  const u32 nDeps = r.ulebc(); const u32 depsOff = r.pos; if (nDeps > 0x07ffffffu) { r.err = KE_SUBARRAY; r.pos = end; } else r.skip32(nDeps * 32);
  const u32 actorLen = r.ulebc(); const u32 actorOff = r.pos; r.skip32(actorLen);
  const u64 seq = r.uleb(), startOp = r.uleb(); (void)r.sleb();
  const u32 msgLen = r.ulebc(); r.skip32(msgLen);
  const u32 nOther = r.ulebc(); const u32 otherOff = r.pos;
  for (u32 i = 0; i < nOther && !r.err; i++) { const u32 l = r.ulebc(); r.skip32(l); }
  const u32 nCols = r.ulebc();
  if (r.err) { o.err = r.err; return; }
  // Column directory and - for single-op changes, the shape of editing traces - the row itself in ONE walk. The data of
  // column k starts at (end of the directory) + (lengths of the columns before it). Checks in the reference's order: column
  // ids ascending over the whole directory (decodeColumnInfo), then per column "no deflated columns" and "bytes present"
  // (decodeChangeColumns).
  const u32 dirPos = r.pos; u32 dataPos = nCols < len ? dirPos + 2 * nCols : end;
  u32 actOff = 0, actLen = 0, pnOff = 0, pnLen = 0, seen = 0, rawLen = 0, keyStrPos = 0, valOff = 0, dirErr = 0; bool haveAct = false, single = false;
  // Fast walk, for what editing traces consist of: a well-formed single-op change whose directory entries are single bytes.
  //  phase A: one pass over the directory; (position, length) of every known column goes to the thread's slot of that
  //           column; anything unusual (multi-byte id / length, deflate bit, ids not ascending, bytes missing) leaves the
  //           fast walk, and the general walk below - the one that knows the reference's error order - starts over;
  //  phase B: the value columns in a fixed order, each decoded by code specialised for it (fast_value); the value
  //           replaces (position, length) in the slot.
  // The fast walk either produces the whole single-op result or nothing.
  bool fastWalk = false;
  if (nCols <= 32 && dirPos + 2 * nCols <= end && len < (1u << 24)) {
    u32 total = 0, bad = 0, nextKey = 0, seenA = 0; bool unk = false;
    for (u32 i = 0; i < nCols; i++) {
      const u32 id = src.ld(dirPos + 2 * i), l = src.ld(dirPos + 2 * i + 1);
      bad |= (id | l) & 0x80u; bad |= id & 8u;
      if (id < nextKey) bad = 1;   // (no deflate bits among accepted ids: the plain compare is the reference's)
      nextKey = id + 1;
      const int ix = slots.index(id & 127u);
      if (ix < 0) unk = true; else { slots.put(ix, ((dataPos + total - off) << 8) | l); seenA |= 1u << ix; }
      total += l;
    }
    if (!bad && !unk && dataPos + total <= end) {   // (a column id this version does not know: the general walk looks at it)
      bool ok = (seenA >> CX_ACTION) & 1u; u32 v = 0;
#define AMG_FAST_COL(IX) if (ok && ((seenA >> IX) & 1u)) { const u32 w = slots.get(IX); if (fast_value<IX>(src, off + (w >> 8), w & 0xffu, v)) slots.put(IX, v); else ok = false; }
      AMG_FAST_COL(CX_ACTION)
      AMG_FAST_COL(CX_OBJ_ACTOR) AMG_FAST_COL(CX_OBJ_CTR) AMG_FAST_COL(CX_KEY_ACTOR) AMG_FAST_COL(CX_KEY_CTR)
      if (ok && ((seenA >> CX_KEY_STR) & 1u)) { const u32 w = slots.get(CX_KEY_STR); keyStrPos = off + (w >> 8) + 2; if (fast_value<CX_KEY_STR>(src, off + (w >> 8), w & 0xffu, v)) slots.put(CX_KEY_STR, v); else ok = false; }
      AMG_FAST_COL(CX_INSERT) AMG_FAST_COL(CX_VAL_LEN) AMG_FAST_COL(CX_PRED_NUM) AMG_FAST_COL(CX_PRED_ACTOR) AMG_FAST_COL(CX_PRED_CTR)
#undef AMG_FAST_COL
      if (ok) {
        if (((seenA >> CX_VAL_RAW) & 1u) && ((seenA >> CX_VAL_LEN) & 1u)) { const u32 w = slots.get(CX_VAL_RAW); valOff = off + (w >> 8); rawLen = w & 0xffu; }
        const u32 pn = (seenA >> CX_PRED_NUM) & 1u ? slots.get(CX_PRED_NUM) : NULL32, predNum = pn == NULL32 ? 0 : pn;
        const u32 vl = (seenA >> CX_VAL_LEN) & 1u ? slots.get(CX_VAL_LEN) : NULL32;
        if (predNum > 1 || (vl == NULL32 ? 0u : (vl >> 4)) > rawLen) ok = false;
        if (predNum == 0 && (seenA & ((1u << CX_PRED_ACTOR) | (1u << CX_PRED_CTR)))) ok = false;
        if (ok) {
          o.h.depsOff = depsOff; o.h.actorOff = actorOff; o.h.actorLen = actorLen; o.h.otherOff = otherOff; o.h.dirOff = dirPos; o.h.dataOff = dataPos;
          o.h.startOp = startOp; o.h.seq = seq;
          o.nDeps = nDeps; o.nOther = nOther; o.nOps = 1; o.nPreds = predNum; o.single = true; o.unknownCols = false;
          o.seen = seenA & ~((1u << CX_VAL_RAW) | (1u << CX_CHLD_ACTOR) | (1u << CX_CHLD_CTR)); o.keyStrPos = (seenA >> CX_KEY_STR) & 1u ? keyStrPos : 0; o.valOff = valOff;
          return;
        }
      }
      keyStrPos = 0; valOff = 0; rawLen = 0;
    }
  }
  if (!fastWalk) {   // general walk: ids / lengths of any size; the end of the directory is guessed (2 bytes per entry) and the walk repeated once with the real one
    o.unknownCols = false;
    for (int attempt = 0; attempt < 2; attempt++) {
      ByteReaderT<S> d(src, dirPos, end); long long lastId = -1; u64 total = 0; u32 colErr = 0; bool orderBad = false, afterValLen = false, groupClash = false;
      single = true; haveAct = false; actLen = pnLen = 0; seen = 0; rawLen = 0; valOff = 0; keyStrPos = 0;
      for (u32 i = 0; i < nCols; i++) {
        const u64 id64 = d.uleb(), l64 = d.uleb();
        if (d.err) break;
        if (lastId >= 0 && ((u32)id64 & ~8u) <= ((u32)lastId & ~8u)) orderBad = true;
        lastId = (long long)id64;
        if (!colErr) { if (id64 & 8) colErr = KE_COL_DEFLATE; else if ((u64)dataPos + total + l64 > (u64)end) colErr = KE_SUBARRAY; }
        const u32 id = id64 > 0xffffffffULL ? 0xffffffffu : (u32)id64, l = (u32)l64, pos = dataPos + (u32)total;
        const int ix = col_index_of(id);
        if (ix < 0) { o.unknownCols = true; if (id64 <= 0xffffffffULL && groups_known_columns(id)) groupClash = true; }
        else {
          if (ix == CX_ACTION) { actOff = (u32)total; actLen = l; haveAct = true; } else if (ix == CX_PRED_NUM) { pnOff = (u32)total; pnLen = l; }
          if (ix == CX_VAL_RAW) { if (afterValLen) { valOff = pos; rawLen = l; } }
          else if (single && !colErr && ix != CX_CHLD_ACTOR && ix != CX_CHLD_CTR) {
            u32 v = 0, used = 0; bool isNull = false;
            if (!single_value(src, ix, pos, l, v, isNull, used)) single = false;
            else { slots.put(ix, isNull ? NULL32 : v); seen |= 1u << ix; if (ix == CX_KEY_STR) keyStrPos = pos + 2; }
          }
        }
        afterValLen = ix == CX_VAL_LEN;
        total += l64;
      }
      if (d.err) { dirErr = d.err; break; }
      if (d.pos != dataPos) { dataPos = d.pos; if (attempt == 0) continue; }   // directory longer than guessed: once more, with its real end
      if (orderBad) dirErr = KE_COL_ORDER; else if (colErr) dirErr = colErr; else if (groupClash) dirErr = KE_GROUP_COLUMN;
      break;
    }
  }
  if (dirErr) { o.err = dirErr; return; }
  u32 predNum = 0;
  if (single) {
    const u32 pn = (seen >> CX_PRED_NUM) & 1u ? slots.get(CX_PRED_NUM) : NULL32; predNum = pn == NULL32 ? 0 : pn;
    const u32 vl = (seen >> CX_VAL_LEN) & 1u ? slots.get(CX_VAL_LEN) : NULL32;
    if (predNum > 1) single = false;
    if ((vl == NULL32 ? 0u : (vl >> 4)) > rawLen) single = false;                                       // the general decoder reports it
    if (predNum == 0 && (seen & ((1u << CX_PRED_ACTOR) | (1u << CX_PRED_CTR)))) single = false;    // pred values without a pred: the general decoder skips them
    if (!haveAct) single = false;
  }
  u32 kerr = 0; u32 nOps = 0; u64 nPreds = 0;
  if (single) { nOps = 1; nPreds = predNum; }
  else {
    nOps = rle_count_values_t(src, dataPos + actOff, dataPos + actOff + actLen, &kerr);
    if (!kerr) nPreds = rle_sum_values_t(src, dataPos + pnOff, dataPos + pnOff + pnLen, nOps, &kerr);
  }
  if (kerr) { o.err = kerr; return; }
  if (nPreds > 0x7fffffffULL || nOps > 0x7fffffffu) { o.err = KE_TOO_LARGE; return; }
  o.h.depsOff = depsOff; o.h.actorOff = actorOff; o.h.actorLen = actorLen; o.h.otherOff = otherOff; o.h.dirOff = dirPos; o.h.dataOff = dataPos;
  o.h.startOp = startOp; o.h.seq = seq;
  o.nDeps = nDeps; o.nOther = nOther; o.nOps = nOps; o.nPreds = (u32)nPreds; o.single = single; o.seen = seen; o.keyStrPos = keyStrPos; o.valOff = valOff;
}
// the row of a single-op change: from the thread's slots to the raw row tables
template <class S> HD void store_single(const ColSlots<S>& slots, const ParsedChange& pc, u32 base, u32 pb, const RawRows& rows) {
  auto val = [&](int ix) -> u32 { return (pc.seen >> ix) & 1u ? slots.get(ix) : NULL32; };
  rows.objActor[base] = val(CX_OBJ_ACTOR); rows.objCtr[base] = val(CX_OBJ_CTR); rows.keyActor[base] = val(CX_KEY_ACTOR); rows.keyCtr[base] = val(CX_KEY_CTR);
  const u32 ksl = val(CX_KEY_STR); rows.keyStrLen[base] = ksl; rows.keyStrOff[base] = ksl == NULL32 ? 0 : pc.keyStrPos;
  rows.insert[base] = (pc.seen >> CX_INSERT) & 1u ? slots.get(CX_INSERT) : 0u; rows.action[base] = val(CX_ACTION);
  rows.valLen[base] = val(CX_VAL_LEN); rows.valOff[base] = pc.valOff; rows.predNum[base] = pc.nPreds; rows.predOff[base] = pb;
  if (pc.nPreds) { rows.predActor[pb] = val(CX_PRED_ACTOR); rows.predCtr[pb] = val(CX_PRED_CTR); }
}
// general expansion of a small change (2 .. SMALL_CHANGE_OPS ops, or one op in a non-canonical encoding): walks the
// directory again and expands every column into rows [base, base + nOps) / preds [pb, pb + nPreds). Returns a KErr.
template <class S> HD u32 expand_change(const S& src, const ChangeHot& h, u32 nOps, u32 nPreds, u32 base, u32 pb, const RawRows& rows) {
  ByteReaderT<S> d(src, h.dirOff, h.dataOff); u32 pos = h.dataOff; u32 seen = 0, kerr = 0;
  while (!d.done()) {
    const u32 id = (u32)d.uleb(), l = (u32)d.uleb(); const int ix = col_index_of(id);
    if (ix >= 0 && ix != CX_VAL_RAW && ix != CX_CHLD_ACTOR && ix != CX_CHLD_CTR) {
      u32 rawOff = 0, rawLen = 0;
      if (ix == CX_VAL_LEN) {   // VALUE_RAW (0x57) directly follows VALUE_LEN (0x56) in the directory when present
        ByteReaderT<S> peek = d; if (!peek.done()) { const u32 nid = (u32)peek.uleb(), nl = (u32)peek.uleb(); if (nid == 0x57) { rawOff = pos + l; rawLen = nl; } }
      }
      const u32 e = decode_one_column_t(src, ix, nOps, base, pos, pos + l, rawOff, rawLen, pb, nPreds, rows);
      if (e && !kerr) kerr = e;
      seen |= 1u << ix;
    }
    pos += l;
  }
  for (int k = 0; k < NCOLS; k++) if (!(seen & (1u << k))) fill_absent_column(k, nOps, base, pb, nPreds, rows);
  return kerr;
}

struct DecodeTilesArgs {
  const u8* arena; const u32* chOff; const u32* chLen; u32 B /* end of the change range of this launch */; u32 first /* its first change */;
  ChangeHot* hot; u32* nOps; u32* nPreds; u32* nDeps; u32* nActors;
  u32* rawBase /* [B] first raw row of each change (every change of the batch) */; u32* rawPredBase /* [B] */;
  u32* decErr /* [B] KErr of the column contents: raised only if the change is applied (the reference decodes columns lazily) */;
  RawRows rows; u32 rowCap, predCap;   // rows are written only inside the capacity; totals[2] tells the host to grow and run again
  unsigned long long* cursor /* [0] ops, [1] preds handed out so far */;
  u32* totals /* [2] overflow [3] bit 0: some change has > SMALL_CHANGE_OPS ops, bit 1: some change has a column with an unknown id; [0] ops and [1] preds are filled from the cursor by k_decode_totals */; u64* errWord; u32 numTiles;
  u32* directList /* [B] changes the staged kernel could not take (outside their tile's staged window) */; u32* directCount /* [1] = CTAs of k_decode_direct that are done */;
  // A launch walks changes first .. B-1 of the batch, perTile per CTA - or, with a list, the changes list[first .. B-1] (the
  // DEFLATEd changes once they are inflated: their bytes lie behind the batch, in list order). A launch without a list leaves
  // out the changes at or behind skipFrom (arena offset): those belong to the list launch.
  const u32* list = nullptr; u32 perTile = 0; u32 skipFrom = 0xffffffffu;
};
// what one thread does with its change once the row range is known
template <class S> HD void finish_change(const DecodeTilesArgs& a, const S& src, const ColSlots<S>& slots, u32 c, const ParsedChange& pc, u32 base, u32 pb) {
  a.hot[c] = pc.h; a.nOps[c] = pc.nOps; a.nPreds[c] = pc.nPreds; a.nDeps[c] = pc.nDeps; a.nActors[c] = 1 + pc.nOther;
  a.rawBase[c] = base; a.rawPredBase[c] = pb;
  u32 kerr = 0;
  if (pc.err) raise(a.errWord, pc.err, c);
  else if (pc.nOps > SMALL_CHANGE_OPS) atomic_or(&a.totals[3], 1u);   // expanded by DecodeColumnKernel once the gate has decided
  else if (pc.nOps > 0) {
    if ((u64)base + pc.nOps > a.rowCap || (u64)pb + pc.nPreds > a.predCap) a.totals[2] = 1;
    else if (pc.single) store_single(slots, pc, base, pb, a.rows);
    else kerr = expand_change(src, pc.h, pc.nOps, pc.nPreds, base, pb, a.rows);
  }
  if (!pc.err && pc.unknownCols) atomic_or(&a.totals[3], 2u);
  a.decErr[c] = kerr;
}

#ifdef AMG_EMU
inline void decode_tiles_begin(Ctx&, const DecodeTilesArgs& a) { a.cursor[0] = a.cursor[1] = 0; a.totals[0] = a.totals[1] = a.totals[2] = a.totals[3] = 0; *a.directCount = 0; }
inline void decode_tiles_range(Ctx& c, DecodeTilesArgs a, u32 first, u32 end) {
  // tiles of 4 changes, last tile first: raw rows are NOT in batch order on the device either (tiles take their row range
  // from a cursor in arrival order), so the emulation makes sure nothing downstream relies on it. DEFLATEd changes wait
  // for the inflate step like on the device (decode_tiles_finish).
  const u32 T = 4, numTiles = (end - first + T - 1) / T;
  for (u32 t = numTiles; t-- > 0;) for (u32 i = first + t * T; i < end && i < first + (t + 1) * T; i++) {
    const u8* p = a.arena + a.chOff[i];
    if (a.chLen[i] > 8 && p[8] == 2 && p[0] == 0x85) { a.directList[(*a.directCount)++] = i; continue; }
    ColSlots<PtrSrc> slots(PtrSrc{a.arena}); ParsedChange pc; parse_change(PtrSrc{a.arena}, slots, a.chOff[i], a.chLen[i], pc);
    if (getenv("AMG_EMU_DECODE_STATS")) { static size_t tot = 0, nonSingle = 0, shown = 0; tot++; if (!pc.single) { nonSingle++; if (shown < 6 && pc.nOps == 1) { shown++; fprintf(stderr, "non-single 1-op change %u:", i); for (u32 k = pc.h.dirOff; k < a.chOff[i] + a.chLen[i]; k++) fprintf(stderr, " %02x", a.arena[k]); fprintf(stderr, "\n"); } } if (tot % 100000 == 0) fprintf(stderr, "decode stats: %zu changes, %zu not single\n", tot, nonSingle); }
    finish_change(a, PtrSrc{a.arena}, slots, i, pc, (u32)std::min<u64>(a.cursor[0], 0x7fffffffu), (u32)std::min<u64>(a.cursor[1], 0x7fffffffu));
    a.cursor[0] += pc.nOps; a.cursor[1] += pc.nPreds;
  }
  c.launches++;
}
inline void decode_tiles_list(Ctx&, DecodeTilesArgs, const u32*, u32, u32 = 32) {}   // (the emulation's range walk lists DEFLATEd changes for the finish step)
inline void decode_tiles_finish(Ctx& c, const DecodeTilesArgs& a, size_t) {
  for (u32 k = 0; k < *a.directCount; k++) {
    const u32 i = a.directList[k];
    ColSlots<PtrSrc> slots(PtrSrc{a.arena}); ParsedChange pc; parse_change(PtrSrc{a.arena}, slots, a.chOff[i], a.chLen[i], pc);
    finish_change(a, PtrSrc{a.arena}, slots, i, pc, (u32)std::min<u64>(a.cursor[0], 0x7fffffffu), (u32)std::min<u64>(a.cursor[1], 0x7fffffffu));
    a.cursor[0] += pc.nOps; a.cursor[1] += pc.nPreds;
  }
  const u64 ops = a.cursor[0], preds = a.cursor[1];
  a.totals[0] = (u32)std::min<u64>(ops, 0x7fffffffu); a.totals[1] = (u32)std::min<u64>(preds, 0x7fffffffu);
  if (ops > a.rowCap || preds > a.predCap) a.totals[2] = 1;   // rows that larger changes reserved must fit as well
  c.launches++;
}
#else
// ---- the tile kernel. One CTA = DT_THREADS consecutive changes of the batch, one thread per change.
//  1. the tile's byte range [lo, hi) of the arena is copied into shared memory by ONE bulk asynchronous copy
//     (cp.async.bulk global -> shared, completion on an mbarrier): every byte of a change crosses HBM -> SM once, in full
//     lines, and the byte-serial parsers below then read shared memory. 8 CTAs are resident per SM, so the copies of some
//     tiles are in flight while others parse. Changes outside their tile's window (inflated changes, which live behind the
//     batch; queue entries; changes too big for the window) are handed to k_decode_direct, which reads global memory.
//  2. every thread parses its change (header, directory, counts; single-op changes keep their row in registers);
//  3. block scan of (ops, preds); the tile takes its raw row range from a global cursor with one atomic (no tile waits for
//     another: a decoupled look-back across 7800 tiles advanced at most 32 tiles per L2 round trip and took 0.5 ms);
//  4. rows are written (single-op: straight from registers, consecutive threads -> consecutive rows; 2..16 ops: second
//     walk over the shared-memory copy); larger changes only reserve their rows.
#ifndef AMG_DT_STAGE_KB
#define AMG_DT_STAGE_KB 19
#endif
#ifndef AMG_DT_MINBLOCKS
#define AMG_DT_MINBLOCKS 8
#endif
static const int DT_THREADS = AMG_DT_THREADS;
static const u32 DT_STAGE = (u32)AMG_DT_STAGE_KB << 10;
DEV u32 smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
DEV u32 sat31(u64 v) { return v > 0x7fffffffULL ? 0x7fffffffu : (u32)v; }
// steps 2-4 for the change of this thread; S = where its bytes are read from
template <class S> DEV void decode_tile_body(const DecodeTilesArgs& a, const S& src, u32 c, bool live, u32 off, u32 len, u64 (*sWarp)[DT_THREADS / 32], u64* sBase) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ColSlots<S> slots(src); ParsedChange pc; pc.nOps = pc.nPreds = 0;
  if (live) parse_change(src, slots, off, len, pc);
  // (ops, preds) of the tile: exclusive scan inside the CTA, 64-bit each (a run-length encoded change can hold 2^31 ops).
  // A warp of single-op changes (the common case) gets its prefixes from two ballots instead of ten shuffles.
  u64 vo = live ? pc.nOps : 0, vp = live ? pc.nPreds : 0; u64 io = vo, ip = vp;
  if (__all_sync(0xffffffffu, vo <= 1 && vp <= 1)) {
    const unsigned le = 0xffffffffu >> (31 - lane);
    io = __popc(__ballot_sync(0xffffffffu, vo == 1) & le); ip = __popc(__ballot_sync(0xffffffffu, vp == 1) & le);
  } else {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const u64 to = __shfl_up_sync(0xffffffffu, io, d), tp = __shfl_up_sync(0xffffffffu, ip, d); if (lane >= d) { io += to; ip += tp; } }
  }
  if (lane == 31) { sWarp[0][warp] = io; sWarp[1][warp] = ip; }
  __syncthreads();
  u64 wo = 0, wp = 0, to = 0, tp = 0;
#pragma unroll
  for (int w = 0; w < DT_THREADS / 32; w++) { const u64 xo = sWarp[0][w], xp = sWarp[1][w]; if (w < warp) { wo += xo; wp += xp; } to += xo; tp += xp; }
  if (tid == 0) {
    // The tile takes its raw row range from a global cursor (one atomic per tile; no tile waits for another). Raw rows are
    // therefore stored in the order in which tiles arrive; FinalizeOpsKernel reads them through rawBase[change], the op
    // order of the batch comes from the scans over the applied changes.
    sBase[0] = atomicAdd(&a.cursor[0], (unsigned long long)to); sBase[1] = tp ? atomicAdd(&a.cursor[1], (unsigned long long)tp) : 0;
  }
  __syncthreads();
  if (live) finish_change(a, src, slots, c, pc, sat31(sBase[0] + wo + io - vo), sat31(sBase[1] + wp + ip - vp));
}
__global__ void __launch_bounds__(DT_THREADS, AMG_DT_MINBLOCKS) k_decode_tiles(const DecodeTilesArgs a) {
  __shared__ __align__(128) u8 stage[DT_STAGE + 16];   // (+16: fast_value may read one byte past a change that ends at the window's end)
  __shared__ __align__(8) unsigned long long bar;
  __shared__ u32 sLo, sHi; __shared__ u64 sWarp[2][DT_THREADS / 32]; __shared__ u64 sBase[2];
  __shared__ u32 sSlots[NCOLS][DT_THREADS]; __shared__ signed char sLut[128];   // ColSlots<SmemSrc>
  const int tid = threadIdx.x, lane = tid & 31;
  for (int k = tid; k < 128; k += DT_THREADS) sLut[k] = (signed char)col_index_of((u32)k);
  if (tid == 0) {
    sLo = 0xffffffffu; sHi = 0;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_addr(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const u32 i = a.first + blockIdx.x * a.perTile + tid; const bool valid = (u32)tid < a.perTile && i < a.B;
  const u32 c = valid ? (a.list ? a.list[i] : i) : 0u;
  u32 off = valid ? a.chOff[c] : 0xffffffffu; const u32 len = valid ? a.chLen[c] : 0;
  bool live = valid && (a.list || off < a.skipFrom);   // (else: a change of the list launch)
  if (!live) off = 0xffffffffu;
  // the staged window starts at the tile's lowest offset; changes that do not lie inside it (a big change may not fit, queue
  // entries may lie anywhere) are passed on to k_decode_direct one by one
  { const u32 lo = __reduce_min_sync(0xffffffffu, off); if (lane == 0) atomicMin(&sLo, lo); }
  __syncthreads();
  const u32 lo16 = sLo & ~15u;
  const bool inWindow = live && (u64)off + len <= (u64)lo16 + DT_STAGE;
  { const u32 hi = __reduce_max_sync(0xffffffffu, inWindow ? off + len : 0u); if (lane == 0 && hi) atomicMax(&sHi, hi); }
  __syncthreads();
  bool defer = live && !inWindow;
  if (defer && !a.list && len > 8 && a.arena[off + 8] == 2 && a.arena[off] == 0x85) defer = false;   // DEFLATEd and outside the window: the list launch takes it, like every DEFLATEd change
  live = inWindow;
  if (sHi > lo16) {
    if (tid == 0) {
      const u32 bytes = ((sHi + 15u) & ~15u) - lo16;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_addr(&bar)), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   :: "r"(smem_addr(stage)), "l"(a.arena + lo16), "r"(bytes), "r"(smem_addr(&bar)) : "memory");
    }
    u32 ok = 0;
    while (!ok) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(smem_addr(&bar)) : "memory");
  }
  const SmemSrc ssrc{smem_addr(stage) - lo16, smem_addr(sLut), smem_addr(&sSlots[0][tid])};
  // DEFLATEd changes (chunk type 2, columnar.js:742) are inflated later in the call and decoded by the list launch then
  const bool deflated = live && len > 8 && ssrc.ld(off + 8) == 2 && ssrc.ld(off) == 0x85;
  if (defer) {
    const unsigned peers = __activemask(); const int leader = __ffs(peers) - 1; u32 base = 0;
    if (lane == leader) base = atomicAdd(a.directCount, (u32)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    a.directList[base + __popc(peers & ((1u << lane) - 1))] = c;
  }
  live = live && !deflated;
  decode_tile_body(a, ssrc, c, live, off, len, sWarp, sBase);
}
// the changes the staged kernel passed on: same steps, one thread per listed change, bytes read from global memory. The last
// CTA to finish turns the cursor into the totals (+ overflow when the reserved rows of larger changes do not fit).
__global__ void __launch_bounds__(DT_THREADS) k_decode_direct(const DecodeTilesArgs a) {
  __shared__ u64 sWarp[2][DT_THREADS / 32]; __shared__ u64 sBase[2];
  const u32 n = *a.directCount;
  for (u32 t = blockIdx.x; t * DT_THREADS < n; t += gridDim.x) {
    const u32 i = t * DT_THREADS + threadIdx.x; const bool live = i < n; const u32 c = live ? a.directList[i] : 0u;
    decode_tile_body(a, PtrSrc{a.arena}, c, live, live ? a.chOff[c] : 0u, live ? a.chLen[c] : 0u, sWarp, sBase);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(a.directCount + 1, 1u) == gridDim.x - 1) {
      const u64 ops = atomicAdd(&a.cursor[0], 0ULL), preds = atomicAdd(&a.cursor[1], 0ULL);
      a.totals[0] = sat31(ops); a.totals[1] = sat31(preds);
      if (ops > a.rowCap || preds > a.predCap) a.totals[2] = 1;
    }
  }
}
// begin (clears cursor / counters) -> any number of ranges (each as soon as its bytes are on the device) -> finish
inline void decode_tiles_begin(Ctx& c, const DecodeTilesArgs& a) {
  CUDA_CHECK(cudaMemsetAsync(a.cursor, 0, 64, c.stream));   // cursor, totals, direct count, done count: one block (Engine::decodeArgs)
}
inline void decode_tiles_range(Ctx& c, DecodeTilesArgs a, u32 first, u32 end) {
  if (end <= first) return;
  a.first = first; a.B = end; a.list = nullptr; a.perTile = DT_THREADS;
  k_decode_tiles<<<(end - first + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, c.stream>>>(a);
  CUDA_CHECK(cudaGetLastError());
  c.launches++;
}
// the inflated changes list[0 .. n): larger than the rest (only changes of 256 bytes and more are compressed), so fewer per tile
inline void decode_tiles_list(Ctx& c, DecodeTilesArgs a, const u32* list, u32 n, u32 perTile = 32) {
  if (n == 0) return;
  a.first = 0; a.B = n; a.list = list; a.perTile = perTile;
  k_decode_tiles<<<(n + perTile - 1) / perTile, DT_THREADS, 0, c.stream>>>(a);
  CUDA_CHECK(cudaGetLastError());
  c.launches++;
}
inline void decode_tiles_finish(Ctx& c, const DecodeTilesArgs& a, size_t numChanges) {
  const size_t tiles = (numChanges + DT_THREADS - 1) / DT_THREADS;
  k_decode_direct<<<(unsigned)std::max<size_t>(1, std::min<size_t>(tiles, (size_t)c.numSMs * 2)), DT_THREADS, 0, c.stream>>>(a);
  CUDA_CHECK(cudaGetLastError());
  c.launches++;
}
#endif

// Changes with more than SMALL_CHANGE_OPS ops: one thread per (column, large change); `large` lists the change indices.
// The column is found by walking the change's directory (at most a few entries).
struct DecodeColumnKernel {
  const u8* arena; const u32* large; size_t numLarge; const ChangeHot* hot; const u32* nOps; const u32* nPreds;
  const u32* rawBase; const u32* rawPredBase; const u8* applied /* per change: decode only if 1 */;
  RawRows rows; u64* errWord; const u32* done /* optional [numLarge][NCOLS]: columns the parallel decoders have expanded already */;
  HD void operator()(size_t t) const {
    const int col = (int)(t / numLarge); const size_t c = large[t % numLarge];
    if (!applied[c]) return;
    if (done && done[(t % numLarge) * NCOLS + col]) return;
    const u32 n = nOps[c]; if (n == 0 || col == CX_VAL_RAW || col == CX_CHLD_ACTOR || col == CX_CHLD_CTR) return;
    const ChangeHot h = hot[c];
    ByteReader d(arena, h.dirOff, h.dataOff); u32 pos = h.dataOff; u32 cOff = 0, cLen = 0, rawOff = 0, rawLen = 0; bool found = false;
    while (!d.done()) {
      const u32 id = (u32)d.uleb(), l = (u32)d.uleb(); const int ix = col_index_of(id);
      if (ix == col) { cOff = pos; cLen = l; found = true; }
      if (ix == CX_VAL_RAW) { rawOff = pos; rawLen = l; }
      pos += l;
    }
    if (!found || cLen == 0) { fill_absent_column(col, n, rawBase[c], rawPredBase[c], nPreds[c], rows); return; }
    const u32 e = decode_one_column(arena, col, n, rawBase[c], cOff, cOff + cLen, rawOff, rawLen, rawPredBase[c], nPreds[c], rows);
    if (e) raise(errWord, e, c);
  }
};
#ifndef AMG_PARSE_MINBLOCKS
#define AMG_PARSE_MINBLOCKS 4
#endif
template <> struct LaunchTraits<ParseKernel> { static const int minBlocks = AMG_PARSE_MINBLOCKS; };
struct LargeFlagKernel { const u32* nOps; const u8* applied; u32* flag; HD void operator()(size_t c) const { flag[c] = (applied[c] && nOps[c] > SMALL_CHANGE_OPS) ? 1u : 0u; } };

}  // namespace amg
