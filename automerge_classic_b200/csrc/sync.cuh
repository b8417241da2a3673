// amgpu — kernels #9: the sync protocol's Bloom filters over the engine's change hashes.
//
// Replaces (reference paths relative to /root/reference):
//   backend/sync.js:38-76   new BloomFilter(hashes): numEntries, 10 bits per entry, 7 probes
//   backend/sync.js:84-111  getProbes / addHash / containsHash (triple hashing over the first 12 digest bytes)
//   backend/sync.js:234-306 makeBloomFilter / getChangesToSend: one probe sequence per candidate change
//
// A candidate is either change i itself (idx == nullptr: every applied change, in application order) or change idx[i].
// Its digest is read straight from Engine::hashes; nothing is rehashed.
#pragma once
#include "gate.cuh"

namespace amg {

static const u32 BLOOM_BITS_PER_ENTRY = 10, BLOOM_NUM_PROBES = 7;   // sync.js:31
static const u32 BLOOM_MAX_PROBES = 64;   // peer filters with more probes are declined (the reference's cost is O(numProbes) per hash)

// x, y, z = little-endian u32 words 0..2 of the digest modulo m (sync.js:88-90); m = 8 * bytes of the filter, 64-bit
HD u64 bloom_word(const u8* h, int k) { return (u64)h[4 * k] | (u64)h[4 * k + 1] << 8 | (u64)h[4 * k + 2] << 16 | (u64)h[4 * k + 3] << 24; }
HD void bloom_seed(const u8* h, u64 m, u64& x, u64& y, u64& z) { x = bloom_word(h, 0) % m; y = bloom_word(h, 1) % m; z = bloom_word(h, 2) % m; }

// sync.js:104-111 addHash: 7 probes into a zeroed bit array. Bit p of the filter is bit (p & 7) of byte p >> 3, which on a
// little-endian device is bit (p & 31) of 32-bit word p >> 5.
struct BloomAddKernel {
  const u8* hashes; const u32* idx; u64 m; u32* bits;
  HD void operator()(size_t i) const {
    const u8* h = hashes + (size_t)(idx ? idx[i] : (u32)i) * 32;
    u64 x, y, z; bloom_seed(h, m, x, y, z);
    for (u32 k = 0; k < BLOOM_NUM_PROBES; k++) {
      if (k) { x = (x + y) % m; y = (y + z) % m; }
      atomic_or(&bits[x >> 5], 1u << (x & 31));
    }
  }
};

// A peer's parsed filter: its bits lie at bitsOff of the uploaded blob. m == 0: the filter contains nothing (no entries, or
// entries but no bits: the reference's NaN probes, sync.js:84-98).
struct BloomRef { u64 bitsOff, m; u32 numProbes, pad; };

// sync.js:273-276: negative[i] = 1 when no filter contains candidate i. A filter contains a hash when all of its
// max(1, numProbes) probes are set (getProbes always yields the first probe).
struct BloomProbeKernel {
  const u8* hashes; const u32* idx; const u8* bits; const BloomRef* filters; u32 numFilters; u8* negative;
  HD void operator()(size_t i) const {
    const u8* h = hashes + (size_t)(idx ? idx[i] : (u32)i) * 32;
    u8 neg = 1;
    for (u32 f = 0; f < numFilters && neg; f++) {
      const BloomRef r = filters[f];
      if (r.m == 0) continue;
      u64 x, y, z; bloom_seed(h, r.m, x, y, z);
      bool all = true;
      for (u32 k = 0; k < (r.numProbes ? r.numProbes : 1u) && all; k++) {
        if (k) { x = (x + y) % r.m; y = (y + z) % r.m; }
        all = (bits[r.bitsOff + (x >> 3)] >> (x & 7)) & 1;
      }
      if (all) neg = 0;
    }
    negative[i] = neg;
  }
};

// out[i] = the digest of change idx[i] (the hashes of the changes a sync message carries)
struct SyncHashGatherKernel {
  const u8* hashes; const u32* idx; u8* out;
  HD void operator()(size_t i) const {
    const u64* s = reinterpret_cast<const u64*>(hashes + (size_t)idx[i] * 32); u64* d = reinterpret_cast<u64*>(out + i * 32);
    d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
  }
};

}  // namespace amg
