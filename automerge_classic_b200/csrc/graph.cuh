// amgpu — kernels #13: hash-graph queries over the engine's change hashes.
//
// Replaces (reference paths relative to /root/reference):
//   backend/new.js:1921-1973  getChanges(haveDeps): the hashes looked up in one launch (HashLookupKernel); the traversals
//                             run on the host over dependency indexes (Engine::changesSince)
//   backend/new.js:1999-2002  getChangeByHash: one lookup
//   backend/new.js:2014-2028  getMissingDeps: the queued changes hashed (ShaKernel) and their dependencies looked up among
//                             the applied and the queued hashes
#pragma once
#include "merge.cuh"

namespace amg {

// The dependency hashes of K parsed changes copied out of their headers (unaligned in the arena) into one dense, 32-byte
// aligned list: change b's j-th dependency goes to out[depBase[b] + j] (the layout HashLookupKernel reads).
struct DepHashCopyKernel {
  const u8* arena; const ChangeMeta* meta; const u32* depBase; u8* out;
  HD void operator()(size_t b) const {
    const ChangeMeta& m = meta[b]; u64* d = reinterpret_cast<u64*>(out + (size_t)depBase[b] * 32);
    for (u32 j = 0; j < m.nDeps; j++)
      for (int k = 0; k < 4; k++) d[4 * j + k] = load_u64_unaligned(arena + m.depsOff + 32 * j + 8 * k);
  }
};

}  // namespace amg
