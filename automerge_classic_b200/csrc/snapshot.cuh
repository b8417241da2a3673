// amgpu — kernels #12: getHistory snapshots. The document after the first k changes of getAllChanges order, filtered from
// the op table the engine keeps (DESIGN.md section 3, "history snapshots").
//
// Replaces (reference paths relative to /root/reference):
//   src/automerge.js:105-118   getHistory's `snapshot` getter: loadChanges(init(), history.slice(0, index + 1)), getPatch
//
// A prefix of getAllChanges order is causally closed, so its document is the current one restricted to the rows and succ
// entries whose op belongs to one of its changes, in the current document order. Every row id and succ entry gets its
// change index once per call (binary search over its actor's changes by maxOp); every prefix length k is then one flag
// pass, two scans and one gather.
#pragma once
#include "history.cuh"

namespace amg {

// change index of op `id`: the change of its actor (changes sorted by (actor, seq): actorStart / changeOrder) with the
// smallest maxOp >= its counter (columnar.js:911-927, as HistAssignKernel)
HD u32 snap_change_of(u64 id, const u32* actorStart, const u32* changeOrder, const long long* cMaxOp, u32 numActors) {
  const u32 a = id_actor(id); const u64 ctr = id_ctr(id);
  if (a >= numActors) return HIST_NONE;
  u32 lo = actorStart[a], hi = actorStart[a + 1]; const u32 end = hi;
  while (lo < hi) { const u32 mid = (lo + hi) >> 1; if ((u64)cMaxOp[changeOrder[mid]] < ctr) lo = mid + 1; else hi = mid; }
  return lo < end ? changeOrder[lo] : HIST_NONE;
}
// one thread per item: ids[i] (a row id or a succ entry) -> its change index; an op outside every change is an error
struct SnapChangeOfKernel {
  const u64* ids; const u32* actorStart; const u32* changeOrder; const long long* cMaxOp; u32 numActors; u32* change; u64* errWord;
  HD void operator()(size_t i) const {
    const u32 k = snap_change_of(ids[i], actorStart, changeOrder, cMaxOp, numActors);
    if (k == HIST_NONE) raise(errWord, KE_HIST_RANGE, i);
    change[i] = k;
  }
};

// one thread per dependency edge e (change j lists change depIdx[e]): firstDep[i] = the smallest j that depends on i
struct SnapFirstDepKernel {
  const u32* depBase; const u32* depIdx; u32 numChanges; u32* firstDep;
  HD void operator()(size_t e) const {
    u32 lo = 0, hi = numChanges;   // owner: the last j with depBase[j] <= e
    while (lo + 1 < hi) { const u32 mid = (lo + hi) >> 1; if (depBase[mid] <= (u32)e) lo = mid; else hi = mid; }
    const u32 d = depIdx[e];
    if (d < numChanges) atomic_min(&firstDep[d], lo);
  }
};

// prefix length k, one thread per row: keep[r] = the row's op is in the prefix; cnt[r] = its succ entries that are
struct SnapKeepKernel {
  const u32* rowChange; const u32* succOff; const u32* succChange; u32 k; u32* keep; u32* cnt;
  HD void operator()(size_t r) const {
    const bool kept = rowChange[r] < k; u32 c = 0;
    if (kept) for (u32 p = succOff[r]; p < succOff[r + 1]; p++) c += succChange[p] < k ? 1u : 0u;
    keep[r] = kept ? 1u : 0u; cnt[r] = c;
  }
};

// prefix length k, one thread per row: a kept row and its kept succ entries (in their order) into the prefix document
struct SnapGatherKernel {
  DocRows d; const u32* succOff; const u64* succ; const u32* succChange; u32 k; u32 N; const u32* keep; const u32* rowPos; const u32* cntPos;
  DocRows o; u32* oSuccOff; u64* oSucc; u32* oSuccCnt;
  HD void operator()(size_t r) const {
    if (r == 0) oSuccOff[rowPos[N]] = cntPos[N];
    if (!keep[r]) return;
    const u32 p = rowPos[r];
    o.id[p] = d.id[r]; o.obj[p] = d.obj[r]; o.key[p] = d.key[r]; o.keyStrOff[p] = d.keyStrOff[r]; o.keyStrLen[p] = d.keyStrLen[r];
    o.flags[p] = d.flags[r]; o.valLen[p] = d.valLen[r]; o.valOff[p] = d.valOff[r]; o.time[p] = d.time[r];
    u32 q = cntPos[r]; oSuccOff[p] = q;
    for (u32 s = succOff[r]; s < succOff[r + 1]; s++) if (succChange[s] < k) oSucc[q++] = succ[s];
    oSuccCnt[p] = q - cntPos[r];
  }
};

// prefix length k, one thread per change i < k: heads (no dependent inside the prefix), clock and maxOp of the prefix
struct SnapHeaderKernel {
  const long long* cActor; const long long* cSeq; const long long* cMaxOp; const u32* firstDep; u32 k; u32 numActors;
  u32* headFlag; unsigned long long* clock; unsigned long long* maxOp;
  HD void operator()(size_t i) const {
    headFlag[i] = firstDep[i] >= k ? 1u : 0u;
    const long long a = cActor[i];
    if (a >= 0 && a < (long long)numActors && cSeq[i] > 0) atomic_max(&clock[a], (unsigned long long)cSeq[i]);
    if (cMaxOp[i] > 0) atomic_max(maxOp, (unsigned long long)cMaxOp[i]);
  }
};

}  // namespace amg
