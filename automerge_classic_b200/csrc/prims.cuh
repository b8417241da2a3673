// amgpu primitives: exclusive scan and stable LSD radix sort (key-value), hand-written for sm_90a.
//
// scan_exclusive : one kernel, decoupled look-back over 2048-element tiles (tile status words tagged with an epoch, so
//                  nothing is cleared between scans; warp 0 inspects 32 predecessor tiles per step). Measured against the
//                  three-kernel form (reduce / scan of tile sums / apply) on the 1M-op trace: 0.1 ms less per call.
// scan_exclusive64: the packed 64-bit scan of the list-index levels keeps the three-kernel form (single pass: no gain).
// radix_sort_pairs: digits of up to 11 bits (balanced over the key width); per pass: tile histogram (shared-memory atomics) -> scan of the
//                  digit-major histogram -> stable scatter. The stable in-tile rank uses
//                  __match_any_sync warp multisplit (one leader lane per digit value per round bumps
//                  a per-warp shared-memory counter), so no sorting network and no second key read.
//                  Only the significant key bits [begin_bit, end_bit) are sorted.
// Both are HBM-bound streaming passes: 4 B (scan) / 12 B (sort) per element read + written per pass.
#pragma once
#include "common.cuh"
#ifdef AMG_EMU
#include <algorithm>
#include <numeric>
#endif

namespace amg {

#ifndef AMG_EMU
// ---------------------------------------------------------------- scan
static const int SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ u32 warp_incl_scan(u32 v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += t; }
  return v;
}
// exclusive scan of one value per thread across a 256-thread CTA; returns exclusive prefix, *total = CTA sum
__device__ __forceinline__ u32 block_excl_scan(u32 v, u32* total, u32* smem /* >= 9 u32 */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u32 incl = warp_incl_scan(v);
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    u32 w = lane < (SCAN_THREADS / 32) ? smem[lane] : 0;
    u32 wi = warp_incl_scan(w);
    if (lane < (SCAN_THREADS / 32)) smem[lane] = wi - w;
    if (lane == (SCAN_THREADS / 32) - 1) smem[8] = wi;
  }
  __syncthreads();
  u32 res = smem[warp] + incl - v;
  *total = smem[8];
  __syncthreads();
  return res;
}

// One launch (decoupled look-back). Tiles take tickets in order; a tile publishes its aggregate, looks back over its
// predecessors (aggregates until the first inclusive prefix) and publishes its own inclusive prefix.
// state word = epoch << 34 | status << 32 | value (status 1 = aggregate, 2 = inclusive prefix).
__global__ void __launch_bounds__(256) k_scan_onepass(const u32* in, u32* out, u64* state, u32* ticket, u32 epoch, size_t n, u32 numTiles) {   // in may alias out
  __shared__ u32 sm[9]; __shared__ u32 sTile, sExcl;
  if (threadIdx.x == 0) sTile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 tile = sTile;
  const size_t base = (size_t)tile * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  u32 v[SCAN_ITEMS]; u32 s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = (base + k < n) ? in[base + k] : 0; s += v[k]; }
  u32 total; u32 ex = block_excl_scan(s, &total, sm);
  if (threadIdx.x < 32) {   // warp 0: publish, look back 32 predecessor tiles at a time, publish again
    volatile u64* st = state; const u64 tag = (u64)epoch << 34; const int lane = threadIdx.x; u32 excl = 0;
    if (lane == 0) st[tile] = tag | ((tile == 0 ? 2ull : 1ull) << 32) | total;
    if (tile > 0) {
      long long p = (long long)tile;
      while (true) {
        const long long idx = p - 1 - lane; u32 status = 2, val = 0;   // before tile 0: an inclusive prefix of zero
        if (idx >= 0) { u64 w; do { w = st[idx]; } while ((w >> 34) != epoch || ((w >> 32) & 3) == 0); status = (u32)(w >> 32) & 3; val = (u32)w; }
        const unsigned inclMask = __ballot_sync(0xffffffffu, status == 2);
        const int first = inclMask ? __ffs(inclMask) - 1 : 32;
        u32 contrib = lane <= first ? val : 0;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, d);
        excl += contrib;
        if (inclMask) break;
        p -= 32;
      }
      if (lane == 0) st[tile] = tag | (2ull << 32) | (u32)(excl + total);
    }
    if (lane == 0) { sExcl = excl; if (tile == numTiles - 1) { out[n] = excl + total; *ticket = 0; } }   // the last ticket holder re-arms the counter
  }
  __syncthreads();
  ex += sExcl;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
}
#endif

struct ScanTemp {
  DBuf<u32> tiles; DBuf<u64> tiles64;
  // single-pass scans (decoupled look-back): per-tile status words tagged with an epoch (no clearing between scans)
  DBuf<u64> state; DBuf<u32> ticket; u32 epoch = 0; size_t stateTiles = 0;
};

#ifndef AMG_EMU
inline void scan_prepare(Ctx& c, ScanTemp& t, size_t numTiles) {   // a fresh epoch; (re)allocation or epoch wrap clears the status words
  if (numTiles + 1 > t.stateTiles || t.epoch >= (1u << 30) - 2) {
    t.stateTiles = numTiles + 1 + numTiles / 2;
    t.state.ensure(c, t.stateTiles); t.ticket.ensure(c, 4);
    dev_memset(c, t.state.p, 0, t.state.cap * 8); dev_memset(c, t.ticket.p, 0, 16); t.epoch = 0;
  }
  t.epoch++;
}
#endif
// out[0..n) = exclusive prefix sums of in[0..n); out[n] = total (out must hold n+1). in == out allowed.
inline void scan_exclusive(Ctx& c, ScanTemp& t, const u32* in, u32* out, size_t n) {
#ifdef AMG_EMU
  u32 acc = 0; for (size_t i = 0; i < n; i++) { u32 v = in[i]; out[i] = acc; acc += v; } out[n] = acc; c.launches += 1;
#else
  if (n == 0) { dev_memset(c, out, 0, sizeof(u32)); return; }
  size_t numTiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  scan_prepare(c, t, numTiles);
  k_scan_onepass<<<(unsigned)numTiles, SCAN_THREADS, 0, c.stream>>>(in, out, t.state.p, t.ticket.p, t.epoch, n, (u32)numTiles);
  CUDA_CHECK(cudaGetLastError());
  c.launches += 1;
#endif
}

// 64-bit variant whose input is produced on the fly by a functor (u64 operator()(size_t i)): used to scan two packed
// 32-bit quantities at once (low word: a count that never overflows 32 bits; high word: a signed sum, mod 2^32).
#ifndef AMG_EMU
__device__ __forceinline__ u64 warp_incl_scan64(u64 v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { u64 t = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += t; }
  return v;
}
__device__ __forceinline__ u64 block_excl_scan64(u64 v, u64* total, u64* smem /* >= 9 */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64 incl = warp_incl_scan64(v);
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    u64 w = lane < (SCAN_THREADS / 32) ? smem[lane] : 0;
    u64 wi = warp_incl_scan64(w);
    if (lane < (SCAN_THREADS / 32)) smem[lane] = wi - w;
    if (lane == (SCAN_THREADS / 32) - 1) smem[8] = wi;
  }
  __syncthreads();
  u64 res = smem[warp] + incl - v;
  *total = smem[8];
  __syncthreads();
  return res;
}
template <class F> __global__ void __launch_bounds__(256) k_scan64_reduce(F in, u64* __restrict__ tileSums, size_t n) {
  __shared__ u64 sm[9];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  u64 s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) if (base + k < n) s += in(base + k);
  u64 total; block_excl_scan64(s, &total, sm);
  if (threadIdx.x == 0) tileSums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(256) k_scan64_tiles(u64* __restrict__ tileSums, size_t numTiles, u64* __restrict__ totalOut) {
  __shared__ u64 sm[9];
  u64 carry = 0;
  for (size_t base = 0; base < numTiles; base += SCAN_THREADS) {
    size_t i = base + threadIdx.x;
    u64 v = i < numTiles ? tileSums[i] : 0, total;
    u64 ex = block_excl_scan64(v, &total, sm);
    if (i < numTiles) tileSums[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) *totalOut = carry;
}
// `tileOffsets` holds exclusive prefix sums of the tile sums (k_scan64_tiles), or - with sumTiles - the raw tile sums,
// which every block then adds up for itself (few tiles: saves the single-block kernel in between)
template <class F> __global__ void __launch_bounds__(256) k_scan64_apply(F in, u64* __restrict__ out, const u64* __restrict__ tileOffsets, size_t n, int sumTiles) {
  __shared__ u64 sm[9];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  u64 offset;
  if (sumTiles) {
    u64 part = 0;
    for (unsigned j = threadIdx.x; j < blockIdx.x; j += SCAN_THREADS) part += tileOffsets[j];
    u64 all; block_excl_scan64(part, &all, sm); offset = all;
  } else offset = tileOffsets[blockIdx.x];
  u64 v[SCAN_ITEMS]; u64 s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = (base + k < n) ? in(base + k) : 0; s += v[k]; }
  u64 total; u64 ex = block_excl_scan64(s, &total, sm) + offset;
  if (sumTiles && blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[n] = offset + total;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
}
#endif
template <class F> inline void scan_exclusive64(Ctx& c, ScanTemp& t, const F& in, u64* out, size_t n) {
#ifdef AMG_EMU
  u64 acc = 0; for (size_t i = 0; i < n; i++) { u64 v = in(i); out[i] = acc; acc += v; } out[n] = acc; c.launches += 2;
#else
  if (n == 0) { dev_memset(c, out, 0, sizeof(u64)); return; }
  size_t numTiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  t.tiles64.ensure(c, numTiles + 1);
  k_scan64_reduce<F><<<(unsigned)numTiles, SCAN_THREADS, 0, c.stream>>>(in, t.tiles64.p, n);
  const bool few = numTiles <= 4096;   // every apply block adds up the tile sums in front of it
  if (!few) k_scan64_tiles<<<1, SCAN_THREADS, 0, c.stream>>>(t.tiles64.p, numTiles, out + n);
  k_scan64_apply<F><<<(unsigned)numTiles, SCAN_THREADS, 0, c.stream>>>(in, out, t.tiles64.p, n, few ? 1 : 0);
  CUDA_CHECK(cudaGetLastError());
  c.launches += few ? 2 : 3;
#endif
}

// ---------------------------------------------------------------- radix sort
#ifndef AMG_EMU
// Digits of up to RS_MAX_BITS bits: a 51-bit sibling key takes 5 passes of 11 bits instead of 7 of 8, a 20-bit field 2 instead
// of 3 (every pass is three launches and a full read + write of the pairs). The digit width of a sort is chosen so that
// its passes are balanced (radix_sort_pairs).
static const int RS_THREADS = 256, RS_ITEMS = 16, RS_TILE = RS_THREADS * RS_ITEMS, RS_WARPS = RS_THREADS / 32, RS_STRIP = 32 * RS_ITEMS, RS_MAX_BITS = 11, RS_MAX_BINS = 1 << RS_MAX_BITS;

__global__ void __launch_bounds__(256) k_rs_hist(const u64* __restrict__ keys, u32* __restrict__ histG, size_t n, int shift, u32 mask, unsigned numTiles) {
  __shared__ u32 hist[RS_MAX_BINS];
  for (u32 k = threadIdx.x; k <= mask; k += RS_THREADS) hist[k] = 0;
  __syncthreads();
  const size_t base = (size_t)blockIdx.x * RS_TILE;
#pragma unroll 4
  for (int j = 0; j < RS_ITEMS; j++) {
    size_t i = base + (size_t)j * RS_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&hist[(u32)(keys[i] >> shift) & mask], 1u);
  }
  __syncthreads();
  for (u32 k = threadIdx.x; k <= mask; k += RS_THREADS) histG[(size_t)k * numTiles + blockIdx.x] = hist[k];
}

__global__ void __launch_bounds__(256) k_rs_scatter(const u64* __restrict__ keysIn, const u32* __restrict__ valsIn, u64* __restrict__ keysOut,
                                                     u32* __restrict__ valsOut, const u32* __restrict__ histScan, size_t n, int shift, u32 mask, unsigned numTiles) {
  __shared__ uint16_t warpHist[RS_WARPS][RS_MAX_BINS];   // a warp's strip holds 512 items: 16-bit counters
  __shared__ u32 digitBase[RS_MAX_BINS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (u32 k = threadIdx.x; k < RS_WARPS * (mask + 1); k += RS_THREADS) warpHist[k / (mask + 1)][k % (mask + 1)] = 0;
  __syncthreads();
  const size_t stripBase = (size_t)blockIdx.x * RS_TILE + (size_t)warp * RS_STRIP;
  u64 key[RS_ITEMS]; u32 val[RS_ITEMS]; u32 rank[RS_ITEMS];
  const u32 ltMask = (1u << lane) - 1u;
#pragma unroll
  for (int j = 0; j < RS_ITEMS; j++) {
    const size_t i = stripBase + (size_t)j * 32 + lane;
    const bool active = i < n;
    key[j] = active ? keysIn[i] : 0; val[j] = active ? valsIn[i] : 0;
    const u32 d = active ? ((u32)(key[j] >> shift) & mask) : 0xffffffffu;
    const u32 peers = __match_any_sync(0xffffffffu, d);
    const int leader = __ffs(peers) - 1;
    u32 base = 0;
    if (active && lane == leader) { base = warpHist[warp][d]; warpHist[warp][d] = (uint16_t)(base + __popc(peers)); }
    base = __shfl_sync(0xffffffffu, base, leader);
    rank[j] = base + __popc(peers & ltMask);
    __syncwarp();
  }
  __syncthreads();
  for (u32 d = threadIdx.x; d <= mask; d += RS_THREADS) {   // per-warp counts of digit d -> exclusive prefixes; + the global base of (digit, tile)
    u32 acc = 0;
#pragma unroll
    for (int w = 0; w < RS_WARPS; w++) { const u32 cnt = warpHist[w][d]; warpHist[w][d] = (uint16_t)acc; acc += cnt; }
    digitBase[d] = histScan[(size_t)d * numTiles + blockIdx.x];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < RS_ITEMS; j++) {
    const size_t i = stripBase + (size_t)j * 32 + lane;
    if (i < n) {
      const u32 d = (u32)(key[j] >> shift) & mask;
      const size_t dst = (size_t)digitBase[d] + warpHist[warp][d] + rank[j];
      keysOut[dst] = key[j]; valsOut[dst] = val[j];
    }
  }
}
#endif

struct SortTemp { DBuf<u32> hist; ScanTemp scan; DBuf<u64> keysAlt; DBuf<u32> valsAlt; };

// Stable sort of (keys, vals) by key bits [beginBit, endBit). `keys`/`vals` are DBufs of size >= n; on
// return they hold the sorted data (the buffers may have been swapped with the temporaries).
inline void radix_sort_pairs(Ctx& c, SortTemp& t, DBuf<u64>& keys, DBuf<u32>& vals, size_t n, int beginBit, int endBit) {
  if (n <= 1 || endBit <= beginBit) return;
#ifdef AMG_EMU
  std::vector<size_t> idx(n); std::iota(idx.begin(), idx.end(), 0);
  const u64 mask = (endBit - beginBit >= 64) ? ~0ULL : (((1ULL << (endBit - beginBit)) - 1) << beginBit);
  std::stable_sort(idx.begin(), idx.end(), [&](size_t a, size_t b) { return (keys.p[a] & mask) < (keys.p[b] & mask); });
  std::vector<u64> k2(n); std::vector<u32> v2(n);
  for (size_t i = 0; i < n; i++) { k2[i] = keys.p[idx[i]]; v2[i] = vals.p[idx[i]]; }
  memcpy(keys.p, k2.data(), n * 8); memcpy(vals.p, v2.data(), n * 4);
  c.launches += 5 * ((endBit - beginBit + 7) / 8);
#else
  const unsigned numTiles = (unsigned)((n + RS_TILE - 1) / RS_TILE);
  const int bits = endBit - beginBit, passes = (bits + RS_MAX_BITS - 1) / RS_MAX_BITS, width = (bits + passes - 1) / passes;   // balanced digit widths
  t.hist.ensure(c, ((size_t)1 << width) * numTiles + 1);
  t.keysAlt.ensure(c, n); t.valsAlt.ensure(c, n);
  for (int shift = beginBit; shift < endBit; shift += width) {
    const int w = std::min(width, endBit - shift); const u32 mask = (1u << w) - 1u;
    k_rs_hist<<<numTiles, RS_THREADS, 0, c.stream>>>(keys.p, t.hist.p, n, shift, mask, numTiles);
    c.launches++;
    scan_exclusive(c, t.scan, t.hist.p, t.hist.p, ((size_t)mask + 1) * numTiles);
    k_rs_scatter<<<numTiles, RS_THREADS, 0, c.stream>>>(keys.p, vals.p, t.keysAlt.p, t.valsAlt.p, t.hist.p, n, shift, mask, numTiles);
    CUDA_CHECK(cudaGetLastError());
    c.launches++;
    std::swap(keys.p, t.keysAlt.p); std::swap(keys.cap, t.keysAlt.cap);
    std::swap(vals.p, t.valsAlt.p); std::swap(vals.cap, t.valsAlt.cap);
  }
#endif
}

}  // namespace amg
