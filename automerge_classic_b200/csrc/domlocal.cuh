// amgpu — list index on the device: the dominance count's global levels in passes of up to DOM_PASS_BITS time bits, and its
// last levels inside shared memory (see DomLevelKernel in patch.cuh for one level).
#pragma once
#include "patch.cuh"
#include "prims.cuh"

namespace amg {
#ifndef AMG_EMU
struct DomLocalBuf { u32 tw[DOM_LOCAL_MAX]; int w[DOM_LOCAL_MAX]; u32 acc[DOM_LOCAL_MAX]; unsigned short gs[DOM_LOCAL_MAX], ge[DOM_LOCAL_MAX]; };
struct DomLocalSmem { DomLocalBuf buf[2]; unsigned short Z[DOM_LOCAL_MAX + 2]; int W[DOM_LOCAL_MAX + 2]; u64 scan[9]; };
__global__ void __launch_bounds__(256) k_dom_local(const DomItem* __restrict__ items, const u32* __restrict__ partHead, const u32* __restrict__ numPartsPtr, u32* __restrict__ qIndex, int bits, u64* errWord) {
  extern __shared__ __align__(16) unsigned char domSmemRaw[];
  DomLocalSmem& S = *reinterpret_cast<DomLocalSmem*>(domSmemRaw);
  const u32 numParts = *numPartsPtr; const int IT = DOM_LOCAL_MAX / 256;
  for (u32 part = blockIdx.x; part < numParts; part += gridDim.x) {
    const u32 g0 = partHead[part]; const u32 m = items[g0].ge - g0;
    if (m > (u32)DOM_LOCAL_MAX) { if (threadIdx.x == 0) raise(errWord, KE_TOO_LARGE, g0); continue; }   // cannot happen (<= 2 items per time)
    for (u32 i = threadIdx.x; i < m; i += 256) { const DomItem it = items[g0 + i]; S.buf[0].tw[i] = it.tw; S.buf[0].w[i] = it.w; S.buf[0].acc[i] = it.acc; S.buf[0].gs[i] = 0; S.buf[0].ge[i] = (unsigned short)m; }
    __syncthreads();
    int cur = 0;
    for (int bit = bits - 1; bit >= 0; bit--) {
      DomLocalBuf& A = S.buf[cur]; DomLocalBuf& B = S.buf[cur ^ 1];
      // exclusive prefix over the items of (bit clear ? 1 : 0) and (bit clear ? weight : 0)
      const u32 lo = threadIdx.x * IT; u64 sum = 0;
      for (int k = 0; k < IT; k++) { const u32 i = lo + k; if (i < m && ((A.tw[i] >> bit) & 1u) == 0) sum += 1ull | ((u64)(u32)A.w[i] << 32); }
      u64 total; u64 ex = block_excl_scan64(sum, &total, S.scan);
      if (threadIdx.x == 0) { S.Z[m] = (unsigned short)(u32)total; S.W[m] = (int)(u32)(total >> 32); }
      for (int k = 0; k < IT; k++) {
        const u32 i = lo + k; if (i >= m) break;
        S.Z[i] = (unsigned short)(u32)ex; S.W[i] = (int)(u32)(ex >> 32);
        if (((A.tw[i] >> bit) & 1u) == 0) ex += 1ull | ((u64)(u32)A.w[i] << 32);
      }
      __syncthreads();
      for (u32 i = threadIdx.x; i < m; i += 256) {
        const u32 tw = A.tw[i]; const u32 gs = A.gs[i], ge = A.ge[i];
        const u32 zg = (u32)S.Z[ge] - (u32)S.Z[gs], zb = (u32)S.Z[i] - (u32)S.Z[gs];
        u32 acc = A.acc[i], dst, ngs = gs, nge = ge;
        if ((tw >> bit) & 1u) { if (dom_query(tw)) acc += (u32)(S.W[i] - S.W[gs]); dst = gs + zg + (i - gs - zb); ngs = gs + zg; }
        else { dst = gs + zb; nge = gs + zg; }
        B.tw[dst] = tw; B.w[dst] = A.w[i]; B.acc[dst] = acc; B.gs[dst] = (unsigned short)ngs; B.ge[dst] = (unsigned short)nge;
      }
      __syncthreads();
      cur ^= 1;
    }
    for (u32 i = threadIdx.x; i < m; i += 256) if (dom_query(S.buf[cur].tw[i])) qIndex[dom_time(S.buf[cur].tw[i]) - 1] = S.buf[cur].acc[i];
    __syncthreads();
  }
}

// ---------------------------------------------------------------- global levels, up to DOM_PASS_BITS time bits per pass
// One pass over time bits [b, b + r) does what r DomLevelKernel levels do: with d = the item's digit (those bits), a query
// adds the weights of the items in front of it in its partition whose digit is smaller, and every partition is split
// stably into 2^r sub-partitions in digit order. k_dom_pass_tile runs the r one-bit levels inside a tile of DOM_PASS_TILE
// items (the partitions cut to the tile, in shared memory); a partition that began in an earlier tile gets the digit counts
// and weights of its earlier items from a decoupled look-back over the tiles (each tile publishes them for the partition
// still open at its end) and the tile that holds a partition's last item knows where each digit's sub-partition starts.
// Items of partitions that go on past their tile wait in `parked` (rank within their digit in place of ge) for
// k_dom_pass_scatter, which reads those starts from the slot of the tile where the partition began (only the partition
// open at a tile's end can start there and go on).
static const int DOM_PASS_BITS = 5, DOM_PASS_TILE = 1024, DOM_PASS_IT = DOM_PASS_TILE / 256;
struct DomPassBuf { u32 acc[DOM_PASS_TILE]; unsigned short src[DOM_PASS_TILE], gs[DOM_PASS_TILE], ge[DOM_PASS_TILE]; };
struct DomPassSmem {
  DomPassBuf buf[2]; u32 tw[DOM_PASS_TILE]; int w[DOM_PASS_TILE]; u32 gs[DOM_PASS_TILE], ge[DOM_PASS_TILE];   // by slot in the tile
  unsigned short Z[DOM_PASS_TILE + 2]; int W[DOM_PASS_TILE + 2]; u64 scan[9];
  u64 carry[32]; u32 carryWBelow[32], firstCnt[32], lastCnt[32], partOff[33]; int firstW[32], lastW[32]; u32 tile;
};
struct DomPassTemp { DBuf<u64> state, agg, incl; DBuf<u32> ticket, slot, parkedFrom; DBuf<DomItem> parked; u32 epoch = 0; size_t tiles = 0; };
__device__ __forceinline__ u64 dom_pair(u32 cnt, int w) { return (u64)cnt | ((u64)(u32)w << 32); }
__global__ void __launch_bounds__(256) k_dom_pass_tile(const DomItem* __restrict__ in, DomItem* __restrict__ out, DomItem* __restrict__ parked, u32* __restrict__ parkedFrom, u32* __restrict__ slot,
                                                       u64* state, u64* agg, u64* incl, u32* ticket, u32 epoch, u32 T, u32 numTiles, int b, int r) {
  __shared__ DomPassSmem S;
  const u32 D = 1u << r, mask = D - 1;
  if (threadIdx.x == 0) S.tile = atomicAdd(ticket, 1u);   // tiles start in ticket order: a tile's predecessors are running
  if (threadIdx.x < 32) { S.firstCnt[threadIdx.x] = S.lastCnt[threadIdx.x] = 0; S.firstW[threadIdx.x] = S.lastW[threadIdx.x] = 0; S.carry[threadIdx.x] = 0; }
  __syncthreads();
  const u32 tile = S.tile, t0 = tile * DOM_PASS_TILE, m = min((u32)DOM_PASS_TILE, T - t0), t1 = t0 + m;
  for (u32 i = threadIdx.x; i < m; i += 256) {
    const DomItem it = in[t0 + i];
    S.tw[i] = it.tw; S.w[i] = it.w; S.gs[i] = it.gs; S.ge[i] = it.ge;
    S.buf[0].acc[i] = it.acc; S.buf[0].src[i] = (unsigned short)i;
    S.buf[0].gs[i] = (unsigned short)(max(it.gs, t0) - t0); S.buf[0].ge[i] = (unsigned short)(min(it.ge, t1) - t0);
  }
  __syncthreads();
  const bool firstCarried = S.gs[0] < t0, lastOpen = S.ge[m - 1] > t1;
  const u32 firstEnd = min(S.ge[0], t1) - t0, lastStart = max(S.gs[m - 1], t0) - t0;
  // digit counts and weights of the first and the last partition piece of the tile
  for (u32 i = threadIdx.x; i < m; i += 256) {
    const u32 d = (S.tw[i] >> b) & mask;
    if (firstCarried && i < firstEnd) { atomicAdd(&S.firstCnt[d], 1u); atomicAdd(&S.firstW[d], S.w[i]); }
    if (lastOpen && i >= lastStart) { atomicAdd(&S.lastCnt[d], 1u); atomicAdd(&S.lastW[d], S.w[i]); }
  }
  __syncthreads();
  // publish the open piece's digit vector, look back for the first piece's carry, publish the inclusive vector (before the
  // levels: the chain of tiles that wait on each other then holds no more than loading and counting)
  if (threadIdx.x < 32) {
    const u32 d = threadIdx.x; volatile u64* st = state; const u64 tag = (u64)epoch << 34;
    const u64 mine = d < D && lastOpen ? dom_pair(S.lastCnt[d], S.lastW[d]) : 0;
    const bool lastIsFirst = lastOpen && firstCarried && lastStart == 0;
    if (!lastIsFirst) incl[(size_t)tile * 32 + d] = mine; else agg[(size_t)tile * 32 + d] = mine;
    __threadfence(); __syncwarp();
    if (d == 0) { __threadfence(); st[tile] = tag | ((lastIsFirst ? 1ull : 2ull) << 32); }
    if (firstCarried) {   // 32 predecessors at a time: their status words, then their vectors up to the first inclusive one
      u64 c = 0;
      for (long long p = (long long)tile; ; p -= 32) {
        const long long q = p - 1 - (long long)d; u32 status = 2;   // (before tile 0: nothing)
        if (q >= 0) { u64 wd; do { wd = st[q]; } while ((wd >> 34) != epoch || ((wd >> 32) & 3) == 0); status = (u32)(wd >> 32) & 3; }
        const unsigned inclMask = __ballot_sync(0xffffffffu, status == 2);
        const int last = inclMask ? __ffs(inclMask) - 1 : 31;
        __threadfence();
        for (int k = 0; k <= last; k++) {
          const u32 sk = __shfl_sync(0xffffffffu, status, k); const long long qk = p - 1 - k;
          if (qk >= 0) c += __ldcg((sk == 2 ? incl : agg) + (size_t)qk * 32 + d);
        }
        if (inclMask) break;
      }
      S.carry[d] = d < D ? c : 0;
      if (lastIsFirst) { incl[(size_t)tile * 32 + d] = c + mine; __threadfence(); __syncwarp(); if (d == 0) { __threadfence(); st[tile] = tag | (2ull << 32); } }
    }
    if (tile == numTiles - 1 && d == 0) *ticket = 0;   // the last ticket re-arms the counter
    __syncwarp();
    // exclusive sums over the digits: carried weights below each digit; where each sub-partition of the first piece's
    // partition starts (when the partition ends in this tile)
    const u32 cc = (u32)S.carry[d], cw = (u32)(S.carry[d] >> 32), hc = cc + S.firstCnt[d];
    u32 exW = cw, exH = hc;
    for (int o = 1; o < 32; o <<= 1) { const u32 a = __shfl_up_sync(0xffffffffu, exW, o), h = __shfl_up_sync(0xffffffffu, exH, o); if (d >= (u32)o) { exW += a; exH += h; } }
    S.carryWBelow[d] = exW - cw; S.partOff[d] = exH - hc;
    if (d == 31) S.partOff[32] = exH;
  }
  __syncthreads();
  // the r one-bit levels on the tile's pieces (k_dom_local's scan + stable split)
  int cur = 0;
  for (int bit = b + r - 1; bit >= b; bit--) {
    DomPassBuf& A = S.buf[cur]; DomPassBuf& B = S.buf[cur ^ 1];
    const u32 lo = threadIdx.x * DOM_PASS_IT; u64 sum = 0;
    for (int k = 0; k < DOM_PASS_IT; k++) { const u32 i = lo + k; if (i < m) { const u32 s = A.src[i]; if (((S.tw[s] >> bit) & 1u) == 0) sum += dom_pair(1, S.w[s]); } }
    u64 total; u64 ex = block_excl_scan64(sum, &total, S.scan);
    if (threadIdx.x == 0) { S.Z[m] = (unsigned short)(u32)total; S.W[m] = (int)(u32)(total >> 32); }
    for (int k = 0; k < DOM_PASS_IT; k++) {
      const u32 i = lo + k; if (i >= m) break;
      S.Z[i] = (unsigned short)(u32)ex; S.W[i] = (int)(u32)(ex >> 32);
      const u32 s = A.src[i]; if (((S.tw[s] >> bit) & 1u) == 0) ex += dom_pair(1, S.w[s]);
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < m; i += 256) {
      const u32 s = A.src[i], tw = S.tw[s], gs = A.gs[i], ge = A.ge[i];
      const u32 zg = (u32)S.Z[ge] - (u32)S.Z[gs], zb = (u32)S.Z[i] - (u32)S.Z[gs];
      u32 acc = A.acc[i], dst, ngs = gs, nge = ge;
      if ((tw >> bit) & 1u) { if (dom_query(tw)) acc += (u32)(S.W[i] - S.W[gs]); dst = gs + zg + (i - gs - zb); ngs = gs + zg; }
      else { dst = gs + zb; nge = gs + zg; }
      B.acc[dst] = acc; B.src[dst] = (unsigned short)s; B.gs[dst] = (unsigned short)ngs; B.ge[dst] = (unsigned short)nge;
    }
    __syncthreads();
    cur ^= 1;
  }
  __syncthreads();
  if (firstCarried && S.ge[0] <= t1 && threadIdx.x <= D) slot[(size_t)(S.gs[0] / DOM_PASS_TILE) * 33 + threadIdx.x] = S.partOff[threadIdx.x];
  if (threadIdx.x == 0) parkedFrom[tile] = lastOpen ? t0 + lastStart : t1;
  const DomPassBuf& F = S.buf[cur];
  for (u32 p = threadIdx.x; p < m; p += 256) {
    const u32 s = F.src[p], tw = S.tw[s], d = (tw >> b) & mask, gs0 = S.gs[s], ge0 = S.ge[s];
    u32 acc = F.acc[p], rank = p - F.gs[p];
    if (gs0 < t0) { rank += (u32)S.carry[d]; if (dom_query(tw)) acc += S.carryWBelow[d]; }
    DomItem o; o.tw = tw; o.w = S.w[s]; o.acc = acc;
    if (ge0 > t1) { o.gs = gs0; o.ge = rank; parked[t0 + p] = o; continue; }
    if (gs0 < t0) { o.gs = gs0 + S.partOff[d]; o.ge = gs0 + S.partOff[d + 1]; out[o.gs + rank] = o; }
    else { o.gs = t0 + F.gs[p]; o.ge = t0 + F.ge[p]; out[t0 + p] = o; }
  }
}
__global__ void __launch_bounds__(256) k_dom_pass_scatter(const DomItem* __restrict__ parked, const u32* __restrict__ parkedFrom, const u32* __restrict__ slot, DomItem* __restrict__ out, u32 T, int b, int r) {
  const u32 mask = (1u << r) - 1;
  for (u32 i = blockIdx.x * 256 + threadIdx.x; i < T; i += gridDim.x * 256) {
    if (i < parkedFrom[i / DOM_PASS_TILE]) continue;
    DomItem o = parked[i];
    const u32* off = slot + (size_t)(o.gs / DOM_PASS_TILE) * 33; const u32 d = (o.tw >> b) & mask, rank = o.ge;
    const u32 gs = o.gs + off[d]; o.ge = o.gs + off[d + 1]; o.gs = gs;
    out[gs + rank] = o;
  }
}
// all global levels: passes of DOM_PASS_BITS bits from the top, the last one narrower; the result is in `items`
inline void dom_global_passes(Ctx& c, DomPassTemp& t, DBuf<DomItem>& items, DBuf<DomItem>& items2, size_t T, int tbits, int localBits) {
  if (T == 0) return;
  const u32 numTiles = (u32)((T + DOM_PASS_TILE - 1) / DOM_PASS_TILE);
  t.parked.ensure(c, T + 1); t.parkedFrom.ensure(c, numTiles + 1); t.slot.ensure(c, (size_t)numTiles * 33 + 1); t.agg.ensure(c, (size_t)numTiles * 32 + 1); t.incl.ensure(c, (size_t)numTiles * 32 + 1);
  for (int hi = tbits; hi > localBits;) {
    const int r = std::min(DOM_PASS_BITS, hi - localBits), b = hi - r;
    if (numTiles + 1 > t.tiles || t.epoch >= (1u << 30) - 2) {   // (re)allocation or epoch wrap: clear the status words
      t.tiles = numTiles + 1 + numTiles / 2; t.state.ensure(c, t.tiles); t.ticket.ensure(c, 4);
      dev_memset(c, t.state.p, 0, t.state.cap * 8); dev_memset(c, t.ticket.p, 0, 16); t.epoch = 0;
    }
    t.epoch++;
    k_dom_pass_tile<<<numTiles, 256, 0, c.stream>>>(items.p, items2.p, t.parked.p, t.parkedFrom.p, t.slot.p, t.state.p, t.agg.p, t.incl.p, t.ticket.p, t.epoch, (u32)T, numTiles, b, r);
    const size_t grid = std::min<size_t>((T + 255) / 256, (size_t)c.numSMs * 8);
    k_dom_pass_scatter<<<(unsigned)grid, 256, 0, c.stream>>>(t.parked.p, t.parkedFrom.p, t.slot.p, items2.p, (u32)T, b, r);
    CUDA_CHECK(cudaGetLastError()); c.launches += 2;
    items.swap(items2); hi = b;
  }
}
#endif

}  // namespace amg
