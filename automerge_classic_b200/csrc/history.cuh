// amgpu — change history of a loaded document: the changes are rebuilt from the document's op table and change metadata.
//
// Replaces (reference paths relative to /root/reference):
//   backend/new.js:1887-1912       computeHashGraph (save -> decodeChanges -> encodeChange per change)
//   backend/columnar.js:876-944    groupChangeOps: preds from succ lists, `del` ops re-synthesised, ops grouped by (actor, maxOp)
//   backend/columnar.js:946-981    decodeDocumentChanges: deps by index -> hashes, hash of every change, heads check
//   backend/columnar.js:132-170, 370-436, 710-738  parseAllOpIds / encodeOps / encodeChange for one change
//
// Shape: sorts and scans build, for every op (document rows + re-synthesised deletions), its change and its sorted pred
// list; one thread per change then encodes its own columns (canonical RLE / delta / boolean records; a change is a few
// ops, and changes are independent) in two passes (size, bytes). A change's bytes contain the hashes of its
// dependencies, so hashing goes level by level through the dependency graph (level = longest path from a root).
// The column writer (hist_column over an op source), the change header writer (write_change_head) and hist_sha256 are
// shared with encodeChanges (encchg.cuh), which reads its ops from a change table instead of the document's rows.
#pragma once
#include "encode.cuh"
#include "prims.cuh"

namespace amg {

static const u32 HIST_NONE = 0xffffffffu;

struct HistI64ToU32Kernel { const long long* in; u32* out; HD void operator()(size_t i) const { out[i] = in[i] == NULLV || in[i] < 0 ? 0u : (u32)in[i]; } };
struct HistIotaKernel { u32* v; HD void operator()(size_t i) const { v[i] = (u32)i; } };
struct HistGatherU32Kernel { const u32* in; const u32* order; u32* out; HD void operator()(size_t j) const { out[j] = in[order[j]]; } };
struct HistPredNumSortedKernel { const u32* opPredNum; const u32* opOrder; u32* out; HD void operator()(size_t j) const { out[j] = opPredNum[opOrder[j]]; } };
struct HistChOffKernel { const u32* outOff; u32 base; u32* chOff; HD void operator()(size_t k) const { chOff[k] = base + outOff[k]; } };
// ---------------------------------------------------------------- preds and deletions from the succ lists
struct HistPairKernel {   // one pair per succ entry: (successor id, predecessor row); pred order key = (counter, actor rank)
  DocRows d; const u32* succOff; const u64* succ; const u32* actorRank; u64* predKey; u64* succKey; u32* pairRow;
  HD void operator()(size_t r) const {
    for (u32 p = succOff[r]; p < succOff[r + 1]; p++) { predKey[p] = (id_ctr(d.id[r]) << 16) | actorRank[id_actor(d.id[r])]; succKey[p] = succ[p]; pairRow[p] = (u32)r; }
  }
};
struct HistGatherKeyKernel { const u64* keyIn; const u32* order; u64* keyOut; HD void operator()(size_t j) const { keyOut[j] = keyIn[order[j]]; } };
struct HistGroupHeadKernel { const u64* key; u32* head; HD void operator()(size_t j) const { head[j] = (j == 0 || key[j] != key[j - 1]) ? 1u : 0u; } };
struct HistIdKeyKernel { DocRows d; u64* key; u32* val; HD void operator()(size_t r) const { key[r] = d.id[r]; val[r] = (u32)r; } };
HD u32 hist_find_row(const u64* sortedIds, const u32* sortedRows, u32 n, u64 id) {
  u32 lo = 0, hi = n;
  while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (sortedIds[mid] < id) lo = mid + 1; else hi = mid; }
  return (lo < n && sortedIds[lo] == id) ? sortedRows[lo] : HIST_NONE;
}
// per successor group g (pairs [start, end)): an existing row gets its pred range, anything else is a deletion
struct HistGroupKernel {
  const u32* head; const u32* groupIdx; const u64* succKeySorted; u32 numPairs; const u64* sortedIds; const u32* sortedRows; u32 numRows;
  u32* groupStart; u64* groupId; u32* groupRow; u32* isDel;
  HD void operator()(size_t j) const {
    if (!head[j]) return;
    const u32 g = groupIdx[j]; groupStart[g] = (u32)j; groupId[g] = succKeySorted[j];
    const u32 row = hist_find_row(sortedIds, sortedRows, numRows, succKeySorted[j]);
    groupRow[g] = row; isDel[g] = row == HIST_NONE ? 1u : 0u;
  }
};
// ops = rows [0, N) then deletions [N, N + numDel): id, a source row (the row itself / one of the deleted rows), pred range
struct HistRowOpKernel { DocRows d; u64* opId; u32* opSrc; u32* opPredStart; u32* opPredNum; HD void operator()(size_t r) const { opId[r] = d.id[r]; opSrc[r] = (u32)r; opPredStart[r] = 0; opPredNum[r] = 0; } };
struct HistGroupOpKernel {
  const u32* groupStart; const u64* groupId; const u32* groupRow; const u32* isDel; const u32* delSlot; const u32* pairRowSorted; u32 numGroups; u32 numPairs; u32 N;
  u64* opId; u32* opSrc; u32* opPredStart; u32* opPredNum;
  HD void operator()(size_t g) const {
    const u32 s = groupStart[g], e = g + 1 < numGroups ? groupStart[g + 1] : numPairs;
    const u32 op = isDel[g] ? N + delSlot[g] : groupRow[g];
    if (isDel[g]) { opId[op] = groupId[g]; opSrc[op] = pairRowSorted[s]; }
    opPredStart[op] = s; opPredNum[op] = e - s;
  }
};
struct HistOpKeyKernel { const u64* opId; u64* key; u32* val; HD void operator()(size_t m) const { key[m] = ((u64)id_actor(opId[m]) << 48) | id_ctr(opId[m]); val[m] = (u32)m; } };

// ---------------------------------------------------------------- ops -> changes
struct HistChangeKeyKernel { const long long* cActor; const long long* cSeq; u64* key; u32* val; HD void operator()(size_t k) const { key[k] = ((u64)cActor[k] << 40) | (u64)cSeq[k]; val[k] = (u32)k; } };
struct HistLowerBoundKernel {   // out[x] = first position whose key is >= (x << shift): segment starts of a sorted key array, gaps included
  const u64* key; u32 n; int shift; u32* out;
  HD void operator()(size_t x) const { const u64 want = (u64)x << shift; u32 lo = 0, hi = n; while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (key[mid] < want) lo = mid + 1; else hi = mid; } out[x] = lo; }
};
// op at sorted position j -> the change of its actor with the smallest maxOp >= counter (columnar.js:911-927)
struct HistAssignKernel {
  const u64* opKey; const u32* actorStart; const u32* changeOrder; const long long* cMaxOp; u32 numActors; int strict; u32* opChange; u64* errWord;
  HD void operator()(size_t j) const {
    const u32 a = (u32)(opKey[j] >> 48); const u64 ctr = opKey[j] & 0xffffffffffffULL;
    if (a >= numActors) { raise(errWord, KE_ACTOR_INDEX, j); opChange[j] = HIST_NONE; return; }
    u32 lo = actorStart[a], hi = actorStart[a + 1];
    const u32 end = hi;
    while (lo < hi) { const u32 mid = (lo + hi) >> 1; if ((u64)cMaxOp[changeOrder[mid]] < ctr) lo = mid + 1; else hi = mid; }
    if (lo >= end) { if (strict) raise(errWord, KE_HIST_RANGE, j); opChange[j] = HIST_NONE; return; }   // not strict: ops of changes applied after the load
    opChange[j] = changeOrder[lo];
  }
};
struct HistChangeStartKernel { const u32* opChange; u32* chOpStart; HD void operator()(size_t j) const { if (opChange[j] != HIST_NONE && (j == 0 || opChange[j] != opChange[j - 1])) chOpStart[opChange[j]] = (u32)j; } };
struct HistChangeCountKernel { const u32* opChange; u32* chNOps; HD void operator()(size_t j) const { if (opChange[j] != HIST_NONE) atomic_add(&chNOps[opChange[j]], 1u); } };
struct HistCheckIdsKernel {   // ids of a change are consecutive and end at its maxOp (columnar.js:929-939)
  const u64* opKey; const u32* opChange; const u32* chOpStart; const u32* chNOps; const long long* cMaxOp; u64* errWord;
  HD void operator()(size_t j) const {
    const u32 k = opChange[j]; const u64 ctr = opKey[j] & 0xffffffffffffULL;
    if (k == HIST_NONE) return;
    const u64 expect = (u64)cMaxOp[k] - chNOps[k] + 1 + ((u32)j - chOpStart[k]);
    if (ctr != expect) raise(errWord, KE_HIST_OPID, j);
  }
};

// ---------------------------------------------------------------- per-change actor tables
// Every op contributes slots for the actors it mentions (object, key element, preds); (change, actor rank) pairs, sorted and
// made unique, are the change's "other actors" in the order encodeChange writes them (sorted by id, author first, columnar.js:154-157)
struct HistOpView {
  DocRows d; const u64* opId; const u32* opSrc; const u32* opPredStart; const u32* opPredNum; const u32* opOrder /* sorted pos -> op */; const u32* pairRowSorted; u32 N;
  HD u32 op(u32 j) const { return opOrder[j]; }
  HD bool isDel(u32 m) const { return m >= N; }
  HD u64 objOf(u32 m) const { return d.obj[opSrc[m]]; }
  HD bool isMapKey(u32 m) const { return d.keyStrLen[opSrc[m]] != NULL32; }
  HD u64 keyElem(u32 m) const {   // list ops: the element the op refers to (0 = _head)
    const u32 r = opSrc[m];
    if (!isDel(m)) return d.key[r];
    return (d.flags[r] & F_INSERT) ? d.id[r] : d.key[r];   // a deletion targets the element its pred row stands for (columnar.js:899-903)
  }
  HD bool insertOf(u32 m) const { return !isDel(m) && (d.flags[opSrc[m]] & F_INSERT); }
  HD u32 actionOf(u32 m) const { return isDel(m) ? (u32)ACT_DEL : flags_action(d.flags[opSrc[m]]); }
  HD u32 valLenOf(u32 m) const { return isDel(m) ? 0u : d.valLen[opSrc[m]]; }
  HD u64 predId(u32 m, u32 i) const { return d.id[pairRowSorted[opPredStart[m] + i]]; }
};
struct HistActorSlotCountKernel { HistOpView v; u32* cnt; HD void operator()(size_t j) const { cnt[j] = 2 + v.opPredNum[v.op((u32)j)]; } };
struct HistActorPairKernel {
  HistOpView v; const u32* slotBase; const u32* opChange; const long long* cActor; const u32* actorRank; u64* key;
  HD u64 mk(u32 k, u32 author, u32 actor) const { return actor == author ? ~0ULL : (((u64)k << 16) | actorRank[actor]); }
  HD void operator()(size_t j) const {
    const u32 m = v.op((u32)j), k = opChange[j]; u32 s = slotBase[j];
    if (k == HIST_NONE) { for (u32 i = 0; i < 2 + v.opPredNum[m]; i++) key[s++] = ~0ULL; return; }
    const u32 author = (u32)cActor[k];
    const u64 obj = v.objOf(m); key[s++] = obj ? mk(k, author, id_actor(obj)) : ~0ULL;
    const u64 ke = v.isMapKey(m) ? 0 : v.keyElem(m); key[s++] = ke ? mk(k, author, id_actor(ke)) : ~0ULL;
    for (u32 i = 0; i < v.opPredNum[m]; i++) key[s++] = mk(k, author, id_actor(v.predId(m, i)));
  }
};
struct HistUniqueKernel { const u64* key; u32* flag; HD void operator()(size_t j) const { flag[j] = (key[j] != ~0ULL && (j == 0 || key[j] != key[j - 1])) ? 1u : 0u; } };
struct HistOtherFillKernel { const u64* key; const u32* flag; const u32* slot; u64* other; HD void operator()(size_t j) const { if (flag[j]) other[slot[j]] = key[j]; } };

// ---------------------------------------------------------------- one change -> bytes
struct ByteSink {
  u8* p; u32 n;
  HD void put(u32 b) { if (p) p[n] = (u8)b; n++; }
  HD void uleb(u64 v) { do { u32 b = v & 0x7f; v >>= 7; if (v) b |= 0x80; put(b); } while (v); }
  HD void sleb(long long v) { while (true) { const u32 b = (u32)(v & 0x7f); const long long rest = v >> 7; const bool done = (rest == 0 && !(b & 0x40)) || (rest == -1 && (b & 0x40)); put(done ? b : (b | 0x80)); if (done) break; v = rest; } }
  HD void bytes(const u8* src, u32 len) { if (p) for (u32 i = 0; i < len; i++) p[n + i] = src[i]; n += len; }
  HD void zeros(u32 len) { if (p) for (u32 i = 0; i < len; i++) p[n + i] = 0; n += len; }
};

// Canonical RLE of the values acc(0..n): maximal runs of equal values; a run of nulls -> [0, n]; a run of >= 2 -> [n, v];
// neighbouring single values -> one literal record [-n, v1..vn]; nothing at all if every value is null (encoding.js:558-783).
template <class Acc> HD void hist_rle(ByteSink& out, const Acc& acc, u32 n) {
  bool any = false; for (u32 i = 0; i < n && !any; i++) any = !acc.isNull(i);
  if (!any) return;
  u32 i = 0;
  while (i < n) {
    if (acc.isNull(i)) { u32 j = i + 1; while (j < n && acc.isNull(j)) j++; out.sleb(0); out.uleb(j - i); i = j; continue; }
    u32 j = i + 1; while (j < n && !acc.isNull(j) && acc.same(i, j)) j++;
    if (j - i >= 2) { out.sleb((long long)(j - i)); acc.put(out, i); i = j; continue; }
    u32 k = i, cnt = 0;
    while (k < n && !acc.isNull(k)) { if (k + 1 < n && !acc.isNull(k + 1) && acc.same(k, k + 1)) break; cnt++; k++; }
    out.sleb(-(long long)cnt); for (u32 t = i; t < i + cnt; t++) acc.put(out, t);
    i += cnt;
  }
}

enum { HC_OBJ_ACTOR, HC_OBJ_CTR, HC_KEY_ACTOR, HC_KEY_CTR, HC_KEY_STR, HC_INSERT, HC_ACTION, HC_VAL_LEN, HC_VAL_RAW, HC_CHLD_ACTOR, HC_CHLD_CTR,
       HC_PRED_NUM, HC_PRED_ACTOR, HC_PRED_CTR, HC_NUM };

// The column writer reads one change's ops through an op source (Src):
//   u32 nOps, nPreds;
//   bool num(int col, u32 i, long long& x)   numeric column value of op i (pred columns: pred i); false = null. Delta
//                                            columns (keyCtr, chldCtr, predCtr) hold the differences already.
//   bool keyNull(u32 i); bool keySame(u32 a, u32 b); void keyPut(ByteSink&, u32 i)   the keyStr column
//   bool insert(u32 i); void valRaw(ByteSink&, u32 i)                              the insert and valRaw columns
// HistChangeCtx is the source over the document's rows (history rebuild), EncChangeSrc (encchg.cuh) the one over a change table.
template <class Src> struct ColNumAcc {   // numeric columns
  const Src& s; int col;
  HD bool isNull(u32 i) const { long long x; return !s.num(col, i, x); }
  HD bool same(u32 a, u32 b) const { long long x = 0, y = 0; s.num(col, a, x); s.num(col, b, y); return x == y; }
  HD void put(ByteSink& out, u32 i) const { long long x = 0; s.num(col, i, x); if (col == HC_KEY_CTR || col == HC_CHLD_CTR || col == HC_PRED_CTR) out.sleb(x); else out.uleb((u64)x); }
};
template <class Src> struct ColStrAcc {   // keyStr
  const Src& s;
  HD bool isNull(u32 i) const { return s.keyNull(i); }
  HD bool same(u32 a, u32 b) const { return s.keySame(a, b); }
  HD void put(ByteSink& out, u32 i) const { s.keyPut(out, i); }
};
// bytes of column `col` of the change (nothing for a column that encodes to nothing)
template <class Src> HD void hist_column(ByteSink& out, const Src& s, int col) {
  switch (col) {
    case HC_KEY_STR: hist_rle(out, ColStrAcc<Src>{s}, s.nOps); break;
    case HC_INSERT: {   // BooleanEncoder (encoding.js:1061-1135): run lengths, starting with false
      bool last = false; u32 cnt = 0;
      for (u32 i = 0; i < s.nOps; i++) { const bool b = s.insert(i); if (b == last) cnt++; else { out.uleb(cnt); last = b; cnt = 1; } }
      if (cnt > 0) out.uleb(cnt);
      break;
    }
    case HC_VAL_RAW: for (u32 i = 0; i < s.nOps; i++) s.valRaw(out, i); break;
    case HC_PRED_ACTOR: case HC_PRED_CTR: hist_rle(out, ColNumAcc<Src>{s, col}, s.nPreds); break;
    default: hist_rle(out, ColNumAcc<Src>{s, col}, s.nOps); break;
  }
}
HD u32 hist_column_id(int col) { const u32 ids[HC_NUM] = {0x01, 0x02, 0x11, 0x13, 0x15, 0x34, 0x42, 0x56, 0x57, 0x61, 0x63, 0x70, 0x71, 0x73}; return ids[col]; }

// The change header (columnar.js:710-739 encodeChange, 659-686 encodeContainer), shared by both encoders. Others writes
// the other actors: n(), put(ByteSink&, q) (length-prefixed id bytes). The dependency hashes are left as zeros: the hash
// kernels write them in sorted order before hashing.
struct ChangeHead { u32 nDeps; const u8* author; u32 authorLen; u64 seq, startOp; long long time; const u8* msg; u32 msgLen; };
template <class Others> HD void change_body_head(ByteSink& b, const ChangeHead& h, const Others& others, const u32* colLen, u32* depsAt) {
  b.uleb(h.nDeps); if (depsAt) *depsAt = b.n; b.zeros(32 * h.nDeps);
  b.uleb(h.authorLen); b.bytes(h.author, h.authorLen); b.uleb(h.seq); b.uleb(h.startOp); b.sleb(h.time); b.uleb(h.msgLen); b.bytes(h.msg, h.msgLen);
  b.uleb(others.n()); for (u32 q = 0; q < others.n(); q++) others.put(b, q);
  u32 nCols = 0; for (int col = 0; col < HC_NUM; col++) if (colLen[col]) nCols++;
  b.uleb(nCols);
  for (int col = 0; col < HC_NUM; col++) if (colLen[col]) { b.uleb(hist_column_id(col)); b.uleb(colLen[col]); }
}
// Container header and body up to the column data into w (a sizing sink writes nothing). Returns the length of the whole
// container (columns and extra bytes included); *depsAt, *bodyAt (the chunk type byte: where the hashed part starts) and
// *dataAt (the first column's bytes) are offsets relative to the container.
template <class Others> HD u32 write_change_head(ByteSink& w, const ChangeHead& h, const Others& others, const u32* colLen, u32 extraLen, u32* depsAt, u32* bodyAt, u32* dataAt) {
  ByteSink s{nullptr, 0}; change_body_head(s, h, others, colLen, nullptr);
  u32 dataLen = 0; for (int col = 0; col < HC_NUM; col++) dataLen += colLen[col];
  const u32 bodyLen = s.n + dataLen + extraLen;
  const u32 start = w.n;
  w.put(0x85); w.put(0x6f); w.put(0x4a); w.put(0x83); w.zeros(4);
  *bodyAt = w.n - start; w.put(1); w.uleb(bodyLen);
  u32 d = 0; change_body_head(w, h, others, colLen, &d); *depsAt = d - start; *dataAt = w.n - start;
  return 8 + 1 + uleb_size(bodyLen) + bodyLen;
}

// everything one change's encoder reads (op source over the document's rows)
struct HistChangeCtx {
  HistOpView v; const u8* arena; u32 k; u32 opStart, nOps, predBase, nPreds;
  const u32* objA; const u32* keyA; const long long* keyDelta; const u32* predA; const long long* predDelta;   // local actor indexes / delta values (HistPrepKernel)
  HD bool num(int col, u32 i, long long& x) const {   // false = null
    if (col == HC_PRED_ACTOR) { x = predA[predBase + i]; return true; }
    if (col == HC_PRED_CTR) { x = predDelta[predBase + i]; return true; }
    const u32 j = opStart + i, m = v.op(j);
    switch (col) {
      case HC_OBJ_ACTOR: if (objA[j] == NULL32) return false; x = objA[j]; return true;
      case HC_OBJ_CTR: { const u64 o = v.objOf(m); if (!o) return false; x = (long long)id_ctr(o); return true; }
      case HC_KEY_ACTOR: if (keyA[j] == NULL32) return false; x = keyA[j]; return true;
      case HC_KEY_CTR: if (keyDelta[j] == NULLV) return false; x = keyDelta[j]; return true;
      case HC_ACTION: x = v.actionOf(m); return true;
      case HC_VAL_LEN: x = v.valLenOf(m); return true;
      case HC_PRED_NUM: x = v.opPredNum[m]; return true;
      default: return false;   // (the document keeps no child columns: always null)
    }
  }
  HD bool keyNull(u32 i) const { return !v.isMapKey(v.op(opStart + i)); }
  HD bool keySame(u32 a, u32 b) const {
    const u32 ra = v.opSrc[v.op(opStart + a)], rb = v.opSrc[v.op(opStart + b)];
    const u32 la = v.d.keyStrLen[ra], lb = v.d.keyStrLen[rb]; if (la != lb) return false;
    const u8* pa = arena + v.d.keyStrOff[ra]; const u8* pb = arena + v.d.keyStrOff[rb];
    for (u32 t = 0; t < la; t++) if (pa[t] != pb[t]) return false;
    return true;
  }
  HD void keyPut(ByteSink& out, u32 i) const { const u32 r = v.opSrc[v.op(opStart + i)]; out.uleb(v.d.keyStrLen[r]); out.bytes(arena + v.d.keyStrOff[r], v.d.keyStrLen[r]); }
  HD bool insert(u32 i) const { return v.insertOf(v.op(opStart + i)); }
  HD void valRaw(ByteSink& out, u32 i) const { const u32 m = v.op(opStart + i); if (!v.isDel(m)) { const u32 r = v.opSrc[m]; out.bytes(arena + v.d.valOff[r], v.d.valLen[r] >> 4); } }
};

struct HistChanges {   // decoded change metadata of the loaded document (one entry per change)
  const long long* actor; const long long* seq; const long long* maxOp; const long long* time; const u32* msgOff; const u32* msgLen;
  const long long* depsNum; const u32* extraOff; const u32* extraLen;
};
// local actor index of a document actor in change k: author 0, others 1 + position in the change's sorted list
HD u32 hist_local_actor(const u64* other, const u32* otherStart, const u32* actorRank, u32 k, u32 author, u32 actor) {
  if (actor == author) return 0;
  const u64 want = ((u64)k << 16) | actorRank[actor];
  u32 lo = otherStart[k], hi = otherStart[k + 1];
  while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (other[mid] < want) lo = mid + 1; else hi = mid; }
  return 1 + (lo - otherStart[k]);
}
// per change: local actor indexes and delta values of its ops and preds, in change order
struct HistPrepKernel {
  HistOpView v; HistChanges ch; const u32* chOpStart; const u32* chNOps; const u32* opPredBase /* per sorted op: first pred slot */; const u64* other; const u32* otherStart; const u32* actorRank;
  u32* objA; u32* keyA; long long* keyDelta; u32* predA; long long* predDelta;
  HD void operator()(size_t k) const {
    const u32 author = (u32)ch.actor[k]; long long keyAbs = 0, predAbs = 0;
    for (u32 i = 0; i < chNOps[k]; i++) {
      const u32 j = chOpStart[k] + i, m = v.op(j);
      const u64 obj = v.objOf(m); objA[j] = obj ? hist_local_actor(other, otherStart, actorRank, (u32)k, author, id_actor(obj)) : NULL32;
      if (v.isMapKey(m)) { keyA[j] = NULL32; keyDelta[j] = NULLV; }
      else {
        const u64 ke = v.keyElem(m);   // 0 = _head: actor null, counter 0 (columnar.js:190-193)
        keyA[j] = ke ? hist_local_actor(other, otherStart, actorRank, (u32)k, author, id_actor(ke)) : NULL32;
        const long long abs = ke ? (long long)id_ctr(ke) : 0; keyDelta[j] = abs - keyAbs; keyAbs = abs;
      }
      for (u32 t = 0; t < v.opPredNum[m]; t++) {
        const u64 pid = v.predId(m, t); const u32 q = opPredBase[j] + t;
        predA[q] = hist_local_actor(other, otherStart, actorRank, (u32)k, author, id_actor(pid));
        const long long abs = (long long)id_ctr(pid); predDelta[q] = abs - predAbs; predAbs = abs;
      }
    }
  }
};
struct HistOthers {   // the other actors of one change: document actors by rank (other: (change << 16 | rank), sorted)
  const u64* other; u32 count; const u32* actorOfRank; const u32* repOff; const u32* repLen; const u8* arena;
  HD u32 n() const { return count; }
  HD void put(ByteSink& b, u32 q) const { const u32 a = actorOfRank[(u32)(other[q] & 0xffff)]; b.uleb(repLen[a]); b.bytes(arena + repOff[a], repLen[a]); }
};
// pass 0: size of the encoded change (container header + body); pass 1: the bytes (dependency hashes left as zeros)
struct HistEncodeKernel {
  int pass; HistOpView v; HistChanges ch; const u8* arena; const u32* chOpStart; const u32* chNOps; const u32* opPredBase; u32 numOpsTotal; u32 numPredsTotal;
  const u64* other; const u32* otherStart; const u32* actorRepOff; const u32* actorRepLen; const u32* actorOfRank /* rank -> actor */;
  const u32* objA; const u32* keyA; const long long* keyDelta; const u32* predA; const long long* predDelta;
  u32* outLen; const u32* outOff; u8* outArena; u32 outBase; u32* depsAt /* per change: arena offset of its dependency hashes */; u32* bodyAt;
  HD void operator()(size_t k) const {
    const u32 opStart = chOpStart[k], nOps = chNOps[k];
    const u32 predBase = nOps ? opPredBase[opStart] : 0;
    const u32 predEnd = nOps ? ((opStart + nOps < numOpsTotal) ? opPredBase[opStart + nOps] : numPredsTotal) : 0;
    HistChangeCtx c{v, arena, (u32)k, opStart, nOps, predBase, predEnd - predBase, objA, keyA, keyDelta, predA, predDelta};
    // column sizes first (the directory precedes the data)
    u32 colLen[HC_NUM];
    for (int col = 0; col < HC_NUM; col++) { ByteSink s{nullptr, 0}; hist_column(s, c, col); colLen[col] = s.n; }
    const u32 author = (u32)ch.actor[k];
    const u32 msgLen = ch.msgLen[k] == NULL32 ? 0 : ch.msgLen[k];
    const ChangeHead h{(u32)ch.depsNum[k], arena + actorRepOff[author], actorRepLen[author], (u64)ch.seq[k], (u64)ch.maxOp[k] - nOps + 1, ch.time[k], arena + ch.msgOff[k], msgLen};
    const HistOthers others{other + otherStart[k], otherStart[k + 1] - otherStart[k], actorOfRank, actorRepOff, actorRepLen, arena};
    ByteSink w{pass ? outArena + outBase + outOff[k] : nullptr, 0};
    u32 dAt = 0, bAt = 0, dataAt = 0;
    const u32 total = write_change_head(w, h, others, colLen, ch.extraLen[k], &dAt, &bAt, &dataAt);
    if (pass == 0) { outLen[k] = total; return; }
    bodyAt[k] = outBase + outOff[k] + bAt; depsAt[k] = outBase + outOff[k] + dAt;
    for (int col = 0; col < HC_NUM; col++) if (colLen[col]) hist_column(w, c, col);
    w.bytes(arena + ch.extraOff[k], ch.extraLen[k]);
  }
};

// ---------------------------------------------------------------- hashes, level by level
HD void hist_sha256(const u8* m, u32 mlen, u8 out[32]) {
#if defined(__CUDA_ARCH__)
  const u32* K = c_sha.k;
#else
  const u32* K = SHA_K;
#endif
  u32 h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  const u32 nBlocks = (mlen + 9 + 63) / 64; u32 w[16];
  for (u32 blk = 0; blk < nBlocks; blk++) {
    const u32 done = blk * 64;
    if (done + 64 <= mlen) {   // full block: 16 independent word loads (as ShaKernel does), not 64 dependent byte loads
      for (int i = 0; i < 16; i++) w[i] = load_be32(m + done + 4 * i);
    } else {
      for (int i = 0; i < 16; i++) {
        u32 x = 0;
        for (int b = 0; b < 4; b++) { const u32 ix = done + 4 * i + b; u32 byte = 0; if (ix < mlen) byte = m[ix]; else if (ix == mlen) byte = 0x80; x = (x << 8) | byte; }
        w[i] = x;
      }
      if (blk == nBlocks - 1) { w[14] = (u32)(((u64)mlen * 8) >> 32); w[15] = (u32)((u64)mlen * 8); }
    }
    sha256_compress(h, w, K);
  }
  for (int i = 0; i < 8; i++) { out[4 * i] = h[i] >> 24; out[4 * i + 1] = h[i] >> 16; out[4 * i + 2] = h[i] >> 8; out[4 * i + 3] = h[i]; }
}
// changes of one level: dependency hashes (of lower levels, so known) written in ascending order, then the change's own hash
struct HistHashKernel {
  const u32* list; u8* arena; const u32* chOff; const u32* chLen; const u32* depsAt; const u32* bodyAt; const long long* depsNum; const u32* depBase; const u32* depIdx; u32 numChanges; u8* hashes; u64* errWord;
  HD void operator()(size_t t) const {
    const u32 k = list[t]; const u32 nd = (u32)depsNum[k]; u8* dst = arena + depsAt[k];
    for (u32 i = 0; i < nd; i++) {   // insertion sort by hash bytes (deps are few)
      const u32 di = depIdx[depBase[k] + i];
      if (di >= numChanges) { raise(errWord, KE_HIST_DEP, k); return; }
      const u8* h = hashes + (size_t)di * 32; u32 pos = i;
      while (pos > 0) { const u8* prev = dst + 32 * (pos - 1); int cmp = 0; for (int b = 0; b < 32 && !cmp; b++) cmp = (int)prev[b] - (int)h[b]; if (cmp <= 0) break; for (int b = 0; b < 32; b++) dst[32 * pos + b] = prev[b]; pos--; }
      for (int b = 0; b < 32; b++) dst[32 * pos + b] = h[b];
    }
    u8 digest[32]; hist_sha256(arena + bodyAt[k], chOff[k] + chLen[k] - bodyAt[k], digest);
    for (int b = 0; b < 32; b++) hashes[(size_t)k * 32 + b] = digest[b];
    for (int b = 0; b < 4; b++) arena[chOff[k] + 4 + b] = digest[b];
  }
};

#ifndef AMG_EMU
// Deep, narrow dependency graphs (one change per actor and level: editing traces) would cost one launch per level. One CTA
// walks a run of consecutive narrow levels instead: the changes of a level in parallel, a barrier between levels (the
// hashes a level reads were written by the same CTA before the barrier).
__global__ void __launch_bounds__(256) k_hist_hash_chain(HistHashKernel hk, const u32* __restrict__ levelStart, u32 firstLevel, u32 numLevels) {
  for (u32 l = 0; l < numLevels; l++) {
    const u32 s = levelStart[firstLevel + l], e = levelStart[firstLevel + l + 1];
    for (u32 t = s + threadIdx.x; t < e; t += 256) hk(t);
    __threadfence();
    __syncthreads();
  }
}
#endif

}  // namespace amg
