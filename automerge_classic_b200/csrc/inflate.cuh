// amgpu — kernels #1b: raw DEFLATE (RFC 1951) decoder, one warp per compressed change.
//
// Replaces (reference paths relative to /root/reference):
//   backend/columnar.js:813-823  inflateChange (pako.inflateRaw on the chunk body of a chunk of type 2)
//
// Changes of 256 bytes and more travel DEFLATEd (columnar.js:738); in the text trace those are the merge changes (many deps),
// about 1 % of the batch and ~300 bytes each; in the nested-map config every change (8 KB). One warp decodes one stream: all lanes
// build the Huffman lookup tables of a block in shared memory, lane 0 walks the symbols (stored, fixed and dynamic blocks).
// Every stream is decoded once, into a scratch area; the sizes lay the inflated changes out behind the batch (prefix sum) and a
// second launch assembles them there (inflate_one).
#pragma once
#include "decode.cuh"

namespace amg {

HD u32 uleb_len(u64 v) { u32 n = 1; while (v >>= 7) n++; return n; }

// ---- decoder with lookup tables (the product path on the device: one warp per stream, tables in shared memory; the
// emulation build runs the same code with a "warp" of one lane). Lane 0 walks the stream; all lanes build the Huffman lookup
// tables of a block: 10 bits for literal / length codes, 8 bits for distance codes (entry = symbol << 4 | code length;
// 0 = code longer than the table: decoded bit by bit from the canonical counts, infl_decode_slow). Configs whose
// changes are all DEFLATEd (C4: 10 000 changes of 8 KB) spent 80 % of a call in the bit-by-bit decoder.
static const int INFL_LBITS = 10, INFL_DBITS = 8, INFL_WARPS = 8;
struct InflWarpTables { uint16_t lit[1 << INFL_LBITS]; uint16_t dist[1 << INFL_DBITS]; uint16_t lcount[16], lsym[288], dcount[16], dsym[32]; u8 lengths[320]; };
#if defined(__CUDA_ARCH__)
#define INFL_SYNC() __syncwarp()
#define INFL_BCAST(x) __shfl_sync(0xffffffffu, (x), 0)
#define INFL_BREV(x) __brev(x)
#else
#define INFL_SYNC() do {} while (0)
#define INFL_BCAST(x) (x)
HD u32 infl_brev_host(u32 v) { u32 r = 0; for (int i = 0; i < 32; i++) { r = (r << 1) | (v & 1u); v >>= 1; } return r; }
#define INFL_BREV(x) infl_brev_host(x)
#endif
struct WarpBits {   // LSB-first bit buffer over src[pos, end)
  const u8* src; u32 pos, end; u64 bb; int bc; bool err;
  HD WarpBits(const u8* s, u32 b, u32 e) : src(s), pos(b), end(e), bb(0), bc(0), err(false) {}
  HD void refill() { while (bc <= 56 && pos < end) { bb |= (u64)src[pos++] << bc; bc += 8; } }
  HD u32 peek(int n) const { return (u32)(bb & ((1ull << n) - 1ull)); }
  HD void drop(int n) { if (n > bc) { err = true; bc = 0; bb = 0; } else { bb >>= n; bc -= n; } }
  HD u32 bits(int n) { if (bc < n) refill(); const u32 v = peek(n); drop(n); return v; }   // n <= 16
  HD void alignByte() { const int r = bc & 7; bb >>= r; bc -= r; }
};
HD int infl_decode_slow(WarpBits& b, const uint16_t* count, const uint16_t* symbol) {   // canonical decode, bit by bit (codes longer than the table)
  int code = 0, first = 0, index = 0;
  for (int len = 1; len < 16; len++) {
    code |= (int)b.bits(1); if (b.err) return -1;
    const int c = count[len];
    if (code - c < first) return symbol[index + (code - first)];
    index += c; first += c; first <<= 1; code <<= 1;
  }
  return -1;
}
// canonical code of n symbols -> count / symbol arrays (lane 0) and the tbits lookup table (all lanes)
HD bool infl_build(const u8* lengths, int n, uint16_t* count, uint16_t* symbol, uint16_t* table, int tbits, int lane, int nlanes, bool mustBeComplete) {
  int ok = 1;
  if (lane == 0) {
    for (int i = 0; i < 16; i++) count[i] = 0;
    for (int i = 0; i < n; i++) count[lengths[i]]++;
    if (count[0] != n) {
      int left = 1;
      for (int len = 1; len < 16; len++) { left <<= 1; left -= count[len]; if (left < 0) { ok = 0; break; } }
      if (ok) {
        uint16_t offs[16]; offs[1] = 0;
        for (int len = 1; len < 15; len++) offs[len + 1] = (uint16_t)(offs[len] + count[len]);
        for (int i = 0; i < n; i++) if (lengths[i]) symbol[offs[lengths[i]]++] = (uint16_t)i;
        ok = (!mustBeComplete || left == 0 || (n - count[0]) == 1) ? 1 : 0;   // (the fixed distance code of RFC 1951 3.2.6 uses 30 of 32 codes)
      }
    }
  }
  ok = INFL_BCAST(ok);
  INFL_SYNC();
  for (int k = lane; k < (1 << tbits); k += nlanes) table[k] = 0;
  INFL_SYNC();
  if (!ok) return false;
  // first canonical code of every length (RFC 1951 3.2.2; count[0] is the number of unused symbols, not a code length)
  u32 next[16]; { u32 code = 0; u32 prev = 0; for (int len = 1; len < 16; len++) { code = (code + prev) << 1; next[len] = code; prev = count[len]; } }
  // symbol[] is sorted by (length, symbol): the j-th symbol of length L has code next[L] + j; codes are sent MSB first into an LSB-first stream
  int base = 0;
  for (int len = 1; len <= tbits; len++) {
    const int c = count[len];
    for (int j = lane; j < c; j += nlanes) {
      const u32 code = next[len] + (u32)j; const u32 rev = INFL_BREV(code) >> (32 - len);
      const uint16_t entry = (uint16_t)((symbol[base + j] << 4) | len);
      for (u32 k = rev; k < (1u << tbits); k += (1u << len)) table[k] = entry;
    }
    base += c;
  }
  INFL_SYNC();
  return true;
}
// Decodes src[begin, end) into dst (nullptr = only count) with the tables T of this warp. Every lane calls it; lane 0
// returns the KErr and *produced.
HD u32 inflate_tabled(InflWarpTables& T, const u8* src, u32 begin, u32 end, u8* dst, u32 dstCap, u32* produced, int lane, int nlanes, u32* softOverflow = nullptr) {
  const uint16_t lenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
  const u8 lenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
  const uint16_t distBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
  const u8 distExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
  const u8 clOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  WarpBits b(src, begin, end); u32 out = 0; u32 e = 0; bool done = false; *produced = 0;
  while (!done && !e) {
    u32 last = 0, type = 0; int nlen = 0, ndist = 0;
    if (lane == 0) {
      last = b.bits(1); type = b.bits(2); if (b.err) e = KE_DEFLATE;
      if (!e && type == 0) {            // stored
        b.alignByte();
        b.pos -= (u32)(b.bc >> 3); b.bb = 0; b.bc = 0;   // the bit buffer holds whole bytes now: given back to the byte position
        if (b.pos + 4 > b.end) e = KE_DEFLATE;
        else {
          const u32 ln = src[b.pos] | ((u32)src[b.pos + 1] << 8), nln = src[b.pos + 2] | ((u32)src[b.pos + 3] << 8);
          if ((ln ^ 0xffffu) != nln) e = KE_DEFLATE;
          else { b.pos += 4; if (b.pos + ln > b.end) e = KE_DEFLATE; else { if (dst && out + ln > dstCap) { if (softOverflow) { *softOverflow = 1; dst = nullptr; } else e = KE_DEFLATE; } if (dst && !e) for (u32 i = 0; i < ln; i++) dst[out + i] = src[b.pos + i]; if (!e) { out += ln; b.pos += ln; } } }
        }
      } else if (!e && type == 1) {     // fixed code (RFC 1951 3.2.6)
        for (int i = 0; i < 144; i++) T.lengths[i] = 8;
        for (int i = 144; i < 256; i++) T.lengths[i] = 9;
        for (int i = 256; i < 280; i++) T.lengths[i] = 7;
        for (int i = 280; i < 288; i++) T.lengths[i] = 8;
        for (int i = 0; i < 30; i++) T.lengths[288 + i] = 5;
        nlen = 288; ndist = 30;
      } else if (!e && type == 2) {     // dynamic code (RFC 1951 3.2.7): the code lengths are decoded by lane 0, bit by bit
        nlen = (int)b.bits(5) + 257; ndist = (int)b.bits(5) + 1; const int ncode = (int)b.bits(4) + 4;
        if (b.err || nlen > 286 || ndist > 30) e = KE_DEFLATE;
        else {
          u8 cl[19]; for (int i = 0; i < 19; i++) cl[i] = 0;
          for (int i = 0; i < ncode; i++) cl[clOrder[i]] = (u8)b.bits(3);
          if (b.err) e = KE_DEFLATE;
          uint16_t* cnt = T.dcount; uint16_t* sym = T.dsym;   // the code-length code (19 symbols) borrows the distance arrays
          for (int i = 0; i < 16; i++) cnt[i] = 0;
          for (int i = 0; i < 19; i++) cnt[cl[i]]++;
          if (!e) {
            if (cnt[0] == 19) { /* no codes: decode fails below */ }
            else {
              int left = 1; for (int l2 = 1; l2 < 16; l2++) { left <<= 1; left -= cnt[l2]; if (left < 0) { e = KE_DEFLATE; break; } }
              if (!e) { uint16_t offs[16]; offs[1] = 0; for (int l2 = 1; l2 < 15; l2++) offs[l2 + 1] = (uint16_t)(offs[l2] + cnt[l2]); for (int i = 0; i < 19; i++) if (cl[i]) sym[offs[cl[i]]++] = (uint16_t)i; if (!(left == 0 || (19 - cnt[0]) == 1)) e = KE_DEFLATE; }
            }
          }
          int idx = 0;
          while (!e && idx < nlen + ndist) {
            const int s2 = infl_decode_slow(b, cnt, sym);
            if (s2 < 0) { e = KE_DEFLATE; break; }
            if (s2 < 16) T.lengths[idx++] = (u8)s2;
            else {
              int rep; u8 val = 0;
              if (s2 == 16) { if (idx == 0) { e = KE_DEFLATE; break; } val = T.lengths[idx - 1]; rep = 3 + (int)b.bits(2); }
              else if (s2 == 17) rep = 3 + (int)b.bits(3);
              else rep = 11 + (int)b.bits(7);
              if (b.err || idx + rep > nlen + ndist) { e = KE_DEFLATE; break; }
              while (rep--) T.lengths[idx++] = val;
            }
          }
          if (!e && T.lengths[256] == 0) e = KE_DEFLATE;   // no end-of-block code
          if (!e) { u8 dl[30]; for (int i = 0; i < ndist; i++) dl[i] = T.lengths[nlen + i]; for (int i = 0; i < ndist; i++) T.lengths[288 + i] = dl[i]; }   // distance lengths at a fixed place
        }
      } else if (!e) e = KE_DEFLATE;
    }
    e = INFL_BCAST(e); type = INFL_BCAST(type); last = INFL_BCAST(last); nlen = INFL_BCAST(nlen); ndist = INFL_BCAST(ndist);
    INFL_SYNC();
    if (e) break;
    if (type != 0) {
      const bool okL = infl_build(T.lengths, nlen, T.lcount, T.lsym, T.lit, INFL_LBITS, lane, nlanes, type == 2);
      const bool okD = infl_build(T.lengths + 288, ndist, T.dcount, T.dsym, T.dist, INFL_DBITS, lane, nlanes, type == 2);
      if (!okL || !okD) { e = KE_DEFLATE; break; }
      if (lane == 0) {
        while (true) {
          b.refill();
          int sym; { const u32 t = T.lit[b.peek(INFL_LBITS)]; if (t) { b.drop((int)(t & 15)); sym = (int)(t >> 4); } else sym = infl_decode_slow(b, T.lcount, T.lsym); }
          if (sym < 0 || b.err) { e = KE_DEFLATE; break; }
          if (sym < 256) { if (dst && out >= dstCap) { if (softOverflow) { *softOverflow = 1; dst = nullptr; } else { e = KE_DEFLATE; break; } } if (dst) dst[out] = (u8)sym; out++; }
          else if (sym == 256) break;
          else {
            sym -= 257; if (sym >= 29) { e = KE_DEFLATE; break; }
            const u32 ln = lenBase[sym] + b.bits(lenExtra[sym]);
            b.refill();
            int ds; { const u32 t = T.dist[b.peek(INFL_DBITS)]; if (t) { b.drop((int)(t & 15)); ds = (int)(t >> 4); } else ds = infl_decode_slow(b, T.dcount, T.dsym); }
            if (ds < 0 || ds >= 30) { e = KE_DEFLATE; break; }
            const u32 d = distBase[ds] + b.bits(distExtra[ds]);
            if (b.err || d > out) { e = KE_DEFLATE; break; }
            if (dst && out + ln > dstCap) { if (softOverflow) { *softOverflow = 1; dst = nullptr; } else { e = KE_DEFLATE; break; } } if (dst) for (u32 i = 0; i < ln; i++) dst[out + i] = dst[out + i - d];
            out += ln;
          }
          if (out > 0x7fffffffu) { e = KE_TOO_LARGE; break; }
        }
      }
      e = INFL_BCAST(e);
      INFL_SYNC();
    }
    if (last) done = true;
  }
  *produced = out;
  return e;
}
// One stream k of the list with `nlanes` cooperating lanes (32 on the device, 1 in the emulation). A stream is decoded ONCE:
//   INFL_SPECULATE: the body goes to scratch[capOff[k] ..) (capacity capOff[k+1] - capOff[k]: a few times the compressed size);
//                   outLen[k] = size of the inflated change (8 bytes magic + checksum, chunk type 1, LEB128 length, body), the
//                   original range is kept in origOff / origLen; a body that does not fit is only counted (ovf[k] = 1);
//   INFL_PLACE:     (after the prefix sum over outLen) the change is assembled at arena[extraStart + outOff[k]): header, then
//                   the body copied from scratch - or, for the few that did not fit, decoded a second time, straight to its place.
enum { INFL_SPECULATE = 0, INFL_PLACE = 1 };
struct InflateArgs {
  u8* arena; u32* chOff; u32* chLen; const u32* list; size_t nd; u32* outLen; const u32* outOff; u32 extraStart; u32* origOff; u32* origLen;
  u8* scratch; const u32* capOff; u32* ovf; u64* errWord;
  u64* total = nullptr;   // INFL_SPECULATE adds every outLen here: each is below 2^31 + 16, so their 32-bit scan wraps for two
};
HD void inflate_one(InflWarpTables& T, size_t k, int pass, const InflateArgs& a, int lane, int nlanes) {
  const u32 c = a.list[k]; const u32 off = pass == INFL_SPECULATE ? a.chOff[c] : a.origOff[k], len = pass == INFL_SPECULATE ? a.chLen[c] : a.origLen[k];
  if (pass == INFL_PLACE && a.outLen[k] == 0) return;
  u32 kerr = 0, streamBegin = 0, clen = 0;
  if (lane == 0) { ByteReader r(a.arena, off + 9, off + len); const u64 cl = r.uleb(); if (r.err || (u64)r.pos + cl > (u64)off + len) kerr = r.err ? r.err : (u32)KE_SUBARRAY; streamBegin = r.pos; clen = (u32)cl; }
  kerr = INFL_BCAST(kerr); streamBegin = INFL_BCAST(streamBegin); clen = INFL_BCAST(clen);
  if (kerr) { if (lane == 0) { raise(a.errWord, kerr, c); if (pass == INFL_SPECULATE) a.outLen[k] = 0; } return; }
  if (pass == INFL_SPECULATE) {
    u8* dst = a.scratch + a.capOff[k]; const u32 cap = a.capOff[k + 1] - a.capOff[k]; u32 out = 0, over = 0;
    const u32 e = inflate_tabled(T, a.arena, streamBegin, streamBegin + clen, dst, cap, &out, lane, nlanes, &over);
    if (lane == 0) {
      if (e) { raise(a.errWord, e, c); a.outLen[k] = 0; }
      else {
        a.outLen[k] = 9 + uleb_len(out) + out; a.origOff[k] = off; a.origLen[k] = len; a.ovf[k] = over;
        if (a.total) atomic_add(reinterpret_cast<unsigned long long*>(a.total), (unsigned long long)a.outLen[k]);
      }
    }
    INFL_SYNC();
    return;
  }
  const u32 total = a.outLen[k];
  u8* d0 = a.arena + a.extraStart + a.outOff[k]; u32 n = 0, hl = 9;
  for (u32 w = 1; w <= 5; w++) { n = total - 9 - w; if (uleb_len(n) == w) break; }
  if (lane == 0) { for (int i = 0; i < 8; i++) d0[i] = a.arena[off + i]; d0[8] = 1; u64 v = n; do { u8 x = v & 0x7f; v >>= 7; if (v) x |= 0x80; d0[hl++] = x; } while (v); }
  hl = INFL_BCAST(hl);
  if (!a.ovf[k]) {
    const u8* body = a.scratch + a.capOff[k];
    for (u32 i = (u32)lane; i < n; i += (u32)nlanes) d0[hl + i] = body[i];
  } else {
    u32 out = 0; const u32 e = inflate_tabled(T, a.arena, streamBegin, streamBegin + clen, d0 + hl, n, &out, lane, nlanes);
    if (lane == 0 && (e || out != n)) raise(a.errWord, e ? e : (u32)KE_DEFLATE, c);
  }
  INFL_SYNC();
}
#ifndef AMG_EMU
__global__ void __launch_bounds__(INFL_WARPS * 32) k_inflate(int pass, const InflateArgs a) {
  __shared__ InflWarpTables tabs[INFL_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (size_t k = (size_t)blockIdx.x * INFL_WARPS + warp; k < a.nd; k += (size_t)gridDim.x * INFL_WARPS) inflate_one(tabs[warp], k, pass, a, lane, 32);
}
#endif
inline void inflate_changes(Ctx& c, int pass, const InflateArgs& a) {
  if (a.nd == 0) return;
#ifdef AMG_EMU
  InflWarpTables* T = new InflWarpTables();
  for (size_t k = 0; k < a.nd; k++) inflate_one(*T, k, pass, a, 0, 1);
  delete T;
#else
  const size_t want = (a.nd + INFL_WARPS - 1) / INFL_WARPS, maxGrid = (size_t)c.numSMs * 4;
  k_inflate<<<(unsigned)std::min(want, maxGrid), INFL_WARPS * 32, 0, c.stream>>>(pass, a);
  CUDA_CHECK(cudaGetLastError());
#endif
  c.launches++;
}
// scratch capacity of a stream: `factor` (four, unless the batch is huge) times its compressed size; a stream that inflates to
// more is decoded a second time, straight into place
struct InflateCapKernel { const u32* list; const u32* chLen; u32 factor; u32* cap; HD void operator()(size_t k) const { cap[k] = factor * chLen[list[k]] + 1024u; } };
// re-points the inflated changes (separate from pass 1: the batch-wide SHA kernel may still be reading the old entries)
struct InflatePatchKernel {
  const u32* list; const u32* outLen; const u32* outOff; u32 extraStart; u32* chOff; u32* chLen;
  HD void operator()(size_t k) const { if (outLen[k] == 0) return; const u32 c = list[k]; chOff[c] = extraStart + outOff[k]; chLen[c] = outLen[k]; }
};
struct DeflateFlagKernel {   // 1 for chunks of type 2 (columnar.js:742); their compressed bytes are summed (scratch sizing)
  const u8* arena; const u32* chOff; const u32* chLen; u32* flag; u32* bytes;
  HD void operator()(size_t c) const { const u8* p = arena + chOff[c]; const bool d = chLen[c] > 8 && p[8] == 2 && p[0] == 0x85; flag[c] = d ? 1u : 0u; warp_agg_add(bytes, d ? chLen[c] : 0u); }
};

}  // namespace amg
