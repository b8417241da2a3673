// amgpu — kernels #12: merge, the changes one document lacks from one or more others, found by hash lookup and copied
// device to device.
//
// Replaces (reference paths relative to /root/reference):
//   backend/new.js:1979-1997  getChangesAdded: which changes of `this` the other document does not have (its
//                             changeIndexByHash lookup, one per change here instead of one per visited hash)
//   src/automerge.js:61-67    merge = applyChanges(local, getChangesAdded(local, remote)): the changes' bytes, gathered
//                             from the remote documents' arenas into one blob the local document applies. Several remotes
//                             share one call: a change two of them hold goes over once, from the first (HashLookupKernel
//                             over a table of the candidates' own hashes, built by HashInsertKernel, which keeps the
//                             smallest position of equal hashes).
#pragma once
#include "gate.cuh"

namespace amg {

// absent[i] = 1 when change i of a source document is not among the target's applied changes (table: the target's hashes)
struct MergeProbeKernel {
  const u8* dstHashes; const u32* table; u64 mask; const u8* srcHashes; u32* absent;
  HD void operator()(size_t i) const { absent[i] = hash_lookup(dstHashes, table, mask, srcHashes + i * 32) == DEP_MISSING ? 1u : 0u; }
};

// idx[i] = the change with digest queries[i] (DEP_MISSING when there is none); queries 8-byte aligned, 32 bytes each
struct HashLookupKernel {
  const u8* hashes; const u32* table; u64 mask; const u8* queries; u32* idx;
  HD void operator()(size_t i) const { idx[i] = hash_lookup(hashes, table, mask, queries + i * 32); }
};

// One change to copy: src[0, len) -> dst[dstOff, dstOff + len), src pointing into the arena of the document that holds the
// change (a merge reads several). dstOff is 64-bit: the blob may pass 4 GiB before the target's arena limit is checked.
struct MergeRange { u64 dstOff; const u8* src; u32 len; };

// One warp per change. When source and destination agree modulo 16, the aligned middle goes as 16-byte words (the
// prefix and the tail byte by byte); otherwise every byte is its own load, still coalesced across the warp.
struct MergeGatherKernel {
  u8* dst; const MergeRange* r;
  struct alignas(16) V16 { u64 a, b; };
  HD void copy(size_t k, u32 lane, u32 lanes) const {
    const MergeRange m = r[k]; const u8* s = m.src; u8* d = dst + m.dstOff; const u64 n = m.len;
    u64 head = n;
    if ((((size_t)s ^ (size_t)d) & 15) == 0) { head = (16 - ((size_t)d & 15)) & 15; if (head > n) head = n; }
    for (u64 i = lane; i < head; i += lanes) d[i] = s[i];
    if (head == n) return;
    const u64 words = (n - head) / 16;
    const V16* sv = reinterpret_cast<const V16*>(s + head); V16* dv = reinterpret_cast<V16*>(d + head);
    for (u64 i = lane; i < words; i += lanes) dv[i] = sv[i];
    for (u64 i = head + words * 16 + lane; i < n; i += lanes) d[i] = s[i];
  }
};

#ifndef AMG_EMU
__global__ void __launch_bounds__(256) k_merge_gather(size_t n, MergeGatherKernel f) {
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t k = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < n; k += warps) f.copy(k, threadIdx.x & 31, 32);
}
#endif
inline void merge_gather(Ctx& c, size_t n, const MergeGatherKernel& f) {
  if (n == 0) return;
#ifdef AMG_EMU
  for (size_t k = 0; k < n; k++) f.copy(k, 0, 1);
#else
  size_t want = (n + 7) / 8, maxGrid = (size_t)c.numSMs * 8;
  k_merge_gather<<<(int)(want < maxGrid ? want : maxGrid), 256, 0, c.stream>>>(n, f);
  CUDA_CHECK(cudaGetLastError());
#endif
  c.launches++;
}

}  // namespace amg
