// amgpu — small glue kernels of the pipeline (flags, compaction, sequence-number check, heads).
#pragma once
#include "patch.cuh"
#include "doccols.cuh"
namespace amg { struct HostChange; }

namespace amg {

// applied[b] = change b is the first copy of its hash and became causally ready (new.js:1555-1586)
struct AppliedFlagKernel {
  const u32* primary; const u32* pass; size_t numApplied; u8* applied; u32* applied32; u32* stats /* [0] count, [1] max finite pass */;
  HD void operator()(size_t b) const {
    const bool a = primary[b] == (u32)(numApplied + b) && pass[b] < PASS_INF;
    applied[b] = a ? 1 : 0; applied32[b] = a ? 1u : 0u;
    warp_agg_add(stats, a ? 1u : 0u); warp_agg_max(stats + 1, a ? pass[b] : 0u);
  }
};
struct PassKeyKernel { const u32* pass; const u8* applied; u64* key; u32* val; HD void operator()(size_t b) const { key[b] = applied[b] ? pass[b] : 0xffffffffu; val[b] = (u32)b; } };
struct RankFromOrderKernel { const u32* order; u32* appRank; size_t numNew; HD void operator()(size_t j) const { if (j < numNew) appRank[order[j]] = (u32)j; } };
struct MaskedCountKernel { const u32* v; const u8* applied; u32* out; HD void operator()(size_t b) const { out[b] = applied[b] ? v[b] : 0u; } };
// general (multi-pass) order: ops of change b start at time 1 + (ops of changes applied before b)
struct OpsInOrderKernel { const u32* nOps; const u8* applied; const u32* appRank; u32* tmp; HD void operator()(size_t b) const { if (applied[b]) tmp[appRank[b]] = nOps[b]; } };
struct TimeBaseKernel { const u32* scanned; const u8* applied; const u32* appRank; const u32* opBase; int inOrder; u32* timeBase; HD void operator()(size_t b) const { timeBase[b] = applied[b] ? (inOrder ? opBase[b] : scanned[appRank[b]]) + 1 : 0; } };
// also raises what the decode kernel found wrong inside the columns of a change that is applied (the reference decodes the
// columns of a change when it applies it, new.js:686-700; a change that stays in the queue is not looked into)
struct MaxOpKernel { const ChangeHot* meta; const u32* nOps; const u8* applied; const u32* decErr; u64* maxOp; u64* errWord; HD void operator()(size_t b) const { u64 v = 0; if (applied[b] && nOps[b] > 0) v = meta[b].startOp + nOps[b] - 1; if (applied[b] && decErr[b]) raise(errWord, decErr[b], b); warp_agg_max(maxOp, v); } };   // one atomic per warp

// amg_debug_decode: raw rows of every change gathered into batch order (predOff re-based to the batch-order pred index)
struct GatherRawKernel {
  size_t numChanges; const u32* opBase; const u32* predBase; const u32* rawBase; const u32* rawPredBase; RawRows raw; u32* out /* [12][M] */; size_t M; u32* predOut /* [2][P] */; size_t P;
  HD void operator()(size_t i) const {
    size_t lo = 0, hi = numChanges; while (hi - lo > 1) { size_t mid = (lo + hi) / 2; if (opBase[mid] <= (u32)i) lo = mid; else hi = mid; }
    const size_t c = lo; const u32 r = rawBase[c] + ((u32)i - opBase[c]);
    const u32* cols[12] = {raw.objActor, raw.objCtr, raw.keyActor, raw.keyCtr, raw.keyStrOff, raw.keyStrLen, raw.insert, raw.action, raw.valLen, raw.valOff, raw.predNum, raw.predOff};
    for (int k = 0; k < 12; k++) out[(size_t)k * M + i] = cols[k][r];
    const u32 po = raw.predOff[r] - rawPredBase[c] + predBase[c]; out[(size_t)11 * M + i] = po;
    for (u32 j = 0; j < raw.predNum[r]; j++) { predOut[po + j] = raw.predActor[raw.predOff[r] + j]; predOut[P + po + j] = raw.predCtr[raw.predOff[r] + j]; }
  }
};
struct RaiseDecErrKernel { const u32* decErr; u64* errWord; HD void operator()(size_t b) const { if (decErr[b]) raise(errWord, decErr[b], b); } };
// new actors: the applied change with the smallest application rank per fresh slot registers the representative bytes
struct NewActorKernel {
  const ChangeHot* meta; const u8* applied; const u32* authorSlot; ActorSlot* slots; u32* newSlots; u32* newCount;
  HD void operator()(size_t b) const {
    if (!applied[b] || authorSlot[b] == EMPTY32) return;
    ActorSlot& s = slots[authorSlot[b]];
    if (s.actorNum != EMPTY32 || (u32)(s.first & 0xffffffffu) != (u32)b) return;
    s.repOff = meta[b].actorOff; s.repLen = meta[b].actorLen;
    newSlots[atomic_add(newCount, 1u)] = authorSlot[b];
  }
};
struct GatherNewActorsKernel {   // slot number, slot record and (up to `stride`) id bytes of every new actor, packed for one copy
  const u8* arena; const ActorSlot* slots; const u32* newSlots; u32* slotOut; ActorSlot* recOut; u8* bytesOut; u32 stride;
  HD void operator()(size_t k) const {
    const u32 s = newSlots[k]; const ActorSlot r = slots[s]; slotOut[k] = s; recOut[k] = r;
    for (u32 j = 0; j < r.repLen && j < stride; j++) bytesOut[k * stride + j] = arena[r.repOff + j];
  }
};
struct SetActorNumKernel { ActorSlot* slots; const u32* slotIds; const u32* nums; HD void operator()(size_t i) const { slots[slotIds[i]].actorNum = nums[i]; } };
struct ChangeActorKernel { const u32* amapBase; const u32* amap; const u8* applied; u32* changeActor; u32* actorCnt; HD void operator()(size_t b) const { if (!applied[b]) { changeActor[b] = EMPTY32; return; } const u32 a = amap[amapBase[b]]; changeActor[b] = a; warp_agg_inc(actorCnt, a); } };
// seq == clock + 1 in application order (new.js:1559, 1571-1579): the seqs of an actor's applied changes must be
// exactly clock+1 .. clock+count, in increasing application order. The change with seq clock+count becomes the actor's
// last applied change: lastChange[a] = its application index (applyLocalChange reads its hash from there).
struct SeqScatterKernel {
  const ChangeHot* meta; const u8* applied; const u32* changeActor; const u32* appRank; const u32* actorBase; const u32* actorCnt; const u64* clock; u32* seqSlot; u32* bad;
  u32* lastChange; u32 numApplied;
  HD void operator()(size_t b) const {
    if (!applied[b]) return;
    const u32 a = changeActor[b]; const u64 seq = meta[b].seq, c0 = clock[a];
    if (seq <= c0 || seq - c0 - 1 >= actorCnt[a]) { *bad = 1; return; }
    if (atomic_cas(&seqSlot[actorBase[a] + (u32)(seq - c0 - 1)], EMPTY32, appRank[b]) != EMPTY32) *bad = 1;
    if (seq - c0 == actorCnt[a]) lastChange[a] = numApplied + appRank[b];
  }
};
struct SeqMonoKernel {
  const ChangeHot* meta; const u8* applied; const u32* changeActor; const u32* actorBase; const u32* actorCnt; const u64* clock; const u32* seqSlot; u32* bad;
  HD void operator()(size_t b) const {
    if (!applied[b]) return;
    const u32 a = changeActor[b]; const u64 seq = meta[b].seq, c0 = clock[a];
    if (seq <= c0 || seq - c0 - 1 >= actorCnt[a]) return;   // out of range: SeqScatterKernel has reported it (and there is no slot to look at)
    const u64 idx = seq - c0 - 1;
    if (idx > 0) { const u32 j = actorBase[a] + (u32)idx; if (seqSlot[j - 1] == EMPTY32 || seqSlot[j - 1] > seqSlot[j]) *bad = 1; }
  }
};
// heads (new.js:1582-1583): every dependency of an applied change stops being a head
struct MarkDepsKernel { const u8* applied; const u32* nDeps; const u32* depBase; const u32* depIdx; u32* isDep; HD void operator()(size_t b) const { if (!applied[b]) return; for (u32 j = 0; j < nDeps[b]; j++) { const u32 d = depIdx[depBase[b] + j]; if (d != DEP_MISSING) isDep[d] = 1; } } };
struct HeadFlag2Kernel { const u8* applied; const u32* isDep; size_t numApplied; u32* flag; HD void operator()(size_t b) const { flag[b] = (applied[b] && !isDep[numApplied + b]) ? 1u : 0u; } };
// The heads of a call travel back in one block of 32-bit words: [0] = number of new heads, [1 .. nOld] = "became a dependency"
// per old head, then per new head (the first `cap` of them) its 32 hash bytes and its rank among the applied changes.
struct HeadsPackKernel {
  const u32* count /* number of new heads */; const u32* list /* their batch indexes */; const u8* batchHashes; const u32* appRank; const u32* isDep; const u32* oldIdx; u32 nOld, cap; u32* out;
  HD void operator()(size_t k) const {
    const u32 nh = *count;
    if (k == 0) out[0] = nh;
    if (k < nOld) out[1 + k] = isDep[oldIdx[k]];
    if (k < cap && k < nh) {
      const u32 b = list[k]; const u32* h = reinterpret_cast<const u32*>(batchHashes + (size_t)b * 32); u32* o = out + 1 + nOld + 9 * k;
      for (int j = 0; j < 8; j++) o[j] = h[j];
      o[8] = appRank[b];
    }
  }
};
struct CompactKernel { const u32* flag; const u32* slot; u32* out; HD void operator()(size_t i) const { if (flag[i]) out[slot[i]] = (u32)i; } };
struct HashGatherKernel { const u8* src; const u8* applied; const u32* appRank; u8* dst; HD void operator()(size_t b) const { if (!applied[b]) return; const u64* s = reinterpret_cast<const u64*>(src + b * 32); u64* d = reinterpret_cast<u64*>(dst + (size_t)appRank[b] * 32); d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3]; } };
// (offset, length) of the changes of a packed batch straight from the caller's offsets array (device copy)
struct OffsetsToRangesKernel { const u64* offsets; u32 shift; u32* off; u32* len; HD void operator()(size_t b) const { off[b] = (u32)offsets[b] + shift; len[b] = (u32)(offsets[b + 1] - offsets[b]); } };
struct SplitPairsKernel { const HostChange* pairs; u32* off; u32* len; HD void operator()(size_t b) const { off[b] = pairs[b].off; len[b] = pairs[b].len; } };
struct PatchPairsKernel { const u32* triples; u32* off; u32* len; HD void operator()(size_t i) const { const u32 c = triples[3 * i]; off[c] = triples[3 * i + 1]; len[c] = triples[3 * i + 2]; } };
// ---------------------------------------------------------------- Backend.load: document chunk -> document table (new.js:1709-1750)
struct DocCountKernel {   // thread 0: number of rows (action column), then sum of succNum
  const u8* arena; DocCols c; u32* out /* [0] rows, [1] succ entries */; u64* errWord;
  HD void operator()(size_t) const {
    u32 err = 0; const u32 n = rle_count_values(arena, c.off[OC_ACTION], c.off[OC_ACTION] + c.len[OC_ACTION], &err);
    u64 s = 0; if (!err) s = rle_sum_values(arena, c.off[OC_SUCC_NUM], c.off[OC_SUCC_NUM] + c.len[OC_SUCC_NUM], n, &err);
    if (err) raise(errWord, err, 0); if (s > 0x7fffffffULL) { raise(errWord, KE_TOO_LARGE, 0); s = 0; }
    out[0] = n; out[1] = (u32)s;
  }
};
struct DocCountRowsKernel {   // rows only; the walk is by record, so a column of a few long runs costs nothing
  const u8* arena; DocCols c; u32* out; u64* errWord;
  HD void operator()(size_t) const { u32 err = 0; out[0] = rle_count_values(arena, c.off[OC_ACTION], c.off[OC_ACTION] + c.len[OC_ACTION], &err); if (err) raise(errWord, err, 0); }
};
struct DocColumnKernel {   // one thread per document column; the change-column decoders are reused through a remapped row view
  const u8* arena; DocCols c; u32 n, numSucc; RawRows rows; u32* idActor; u32* idCtr; u64* errWord; u32 mask /* columns to decode here */;
  HD void operator()(size_t k) const {
    const int col = doc_col_decoder((int)k);
    if (!((mask >> k) & 1u) || col < 0) return;
    const RawRows r = doc_col_rows((int)k, rows, idActor, idCtr);
    u32 e;
    if (c.len[k] == 0) { fill_absent_column(col, n, 0, 0, numSucc, r); e = 0; }
    else e = decode_one_column(arena, col, n, 0, c.off[k], c.off[k] + c.len[k], c.off[OC_VAL_RAW], c.len[OC_VAL_RAW], 0, numSucc, r);
    if (e) raise(errWord, e, k);
  }
};
// utf8 key column of a long document: one thread walks the records (a repetition or a null run is one step whatever its
// length; only literal strings are visited one by one), every row then looks its record up. Same reader, same errors.
struct DocKeyStrRecordsKernel {
  const u8* arena; u32 off, len, n; u32* recStart; u32* recStrOff; u32* recStrLen; u32* numRecOut /* [0] records, [1] values covered */; u64* errWord;
  HD void operator()(size_t) const {
    RleReader a(arena, off, off + len, 2); u32 seen = 0, R = 0;
    while (!a.done() && !a.r.err && seen < n) {
      long long v; u32 o = 0, l = 0; const bool nn = a.next(v, o, l);
      if (a.r.err) break;
      u64 adv = 1;
      if (a.state != 2 && a.count > 0) { adv += (u64)a.count; a.count = 0; }
      if (seen + adv > n) adv = n - seen;
      recStart[R] = seen; recStrOff[R] = nn ? o : 0; recStrLen[R] = nn ? l : NULL32; R++;
      seen += (u32)adv;
    }
    if (a.r.err) raise(errWord, a.r.err, 4);
    if (seen < n) { recStart[R] = seen; recStrOff[R] = 0; recStrLen[R] = NULL32; R++; }   // a reader past the end of the column yields null
    recStart[R] = n; numRecOut[0] = R; numRecOut[1] = seen;
  }
};
struct DocKeyStrExpandKernel {
  const u32* recStart; const u32* recStrOff; const u32* recStrLen; u32 R; u32* keyStrOff; u32* keyStrLen;
  HD void operator()(size_t i) const {
    u32 lo = 0, hi = R;
    while (hi - lo > 1) { const u32 mid = (lo + hi) >> 1; if (recStart[mid] <= (u32)i) lo = mid; else hi = mid; }
    keyStrOff[i] = recStrOff[lo]; keyStrLen[i] = recStrLen[lo];
  }
};
// clock of a long loaded document (new.js:1645-1675 readDocumentChanges): changes sorted by actor (stable), every change
// compared with the same actor's previous one
struct ClockKeyKernel { const long long* actor; u32 numActors; u64* key; u32* val; u32* bad; HD void operator()(size_t i) const { const long long a = actor[i]; if (a == NULLV || a < 0 || (u64)a >= numActors) { *bad = 1; key[i] = 0; } else key[i] = (u64)a; val[i] = (u32)i; } };
struct ClockCheckKernel {   // (lastChange: the index of each actor's last change)
  const u64* key; const u32* val; const long long* seq; u32 n; u64* clock; u32* bad; u32* lastChange;
  HD void operator()(size_t j) const {
    const u32 i = val[j]; const long long s = seq[i] == NULLV ? 0 : seq[i];
    const bool havePrev = j > 0 && key[j - 1] == key[j];
    const long long ps = havePrev ? (seq[val[j - 1]] == NULLV ? 0 : seq[val[j - 1]]) : 0;
    if (!(s == 1 || (havePrev && s == ps + 1)) || s < 0) *bad = 1;
    if (j + 1 == n || key[j + 1] != key[j]) { clock[key[j]] = (u64)s; lastChange[key[j]] = i; }
  }
};
struct DocAbsentKernel {   // fill_absent_column for a long document, one thread per row (col as in DocColumnKernel, rows from doc_col_rows)
  int col; RawRows r;
  HD void operator()(size_t i) const { fill_absent_column(col, 1, (u32)i, col == CX_PRED_NUM ? 0u : (u32)i, 1, r); }   // row i (pred columns: entry i); an absent succNum gives offset 0
};
struct DebugColumnKernel {   // amg_debug_decode_column, serial side: the readers of the load path on one column
  int kind; const u8* bytes; u32 len; u32 n; long long* out; u32* tmp; u64* errWord;
  HD void operator()(size_t) const {
    u32 kerr = 0;
    if (kind == 3) {
      RawRows rr; memset(&rr, 0, sizeof(rr)); rr.insert = tmp;
      kerr = decode_one_column(bytes, CX_INSERT, n, 0, 0, len, 0, 0, 0, 0, rr);
      for (u32 i = 0; i < n; i++) out[i] = tmp[i];
    } else {
      RleReader r(bytes, 0, len, kind == 0 ? 0 : 1); long long acc = 0;
      for (u32 i = 0; i < n; i++) {
        long long v = 0; u32 o, l; const bool nn = r.next(v, o, l);
        if (!nn) { out[i] = NULLV; continue; }
        if (kind == 2) { acc += v; out[i] = acc; } else out[i] = v;
      }
      kerr = r.r.err;
    }
    if (kerr) raise(errWord, kerr, 0);
  }
};
struct U32ToI64Kernel { const u32* in; long long* out; HD void operator()(size_t i) const { out[i] = in[i]; } };
struct DocFinalizeKernel {
  RawRows raw; const u32* idActor; const u32* idCtr; u32 numActors; DocRows d; u32* succOff; u64* succ; u64* maxOp; u64* errWord;
  HD void operator()(size_t i) const {
    bool bad = false;
    auto actor = [&](u32 a) -> u32 { if (a >= numActors) { bad = true; return 0; } return a; };
    d.id[i] = pack_id(idCtr[i], actor(idActor[i]));
    const u32 oa = raw.objActor[i], oc = raw.objCtr[i];
    d.obj[i] = (oc == NULL32 || oa == NULL32) ? 0 : pack_id(oc, actor(oa));
    const u32 ka = raw.keyActor[i], kc = raw.keyCtr[i];
    d.key[i] = (kc == NULL32 || kc == 0 || ka == NULL32) ? 0 : pack_id(kc, actor(ka));
    d.keyStrOff[i] = raw.keyStrOff[i]; d.keyStrLen[i] = raw.keyStrLen[i];
    const u32 act = raw.action[i];
    d.flags[i] = (raw.insert[i] ? F_INSERT : 0) | ((act == NULL32 ? 0xffffu : (act > 0xfffe ? 0xfffeu : act)) << 8);
    d.valLen[i] = raw.valLen[i] == NULL32 ? 0 : raw.valLen[i]; d.valOff[i] = raw.valOff[i]; d.time[i] = 0;
    succOff[i] = raw.predOff[i];
    u64 mx = idCtr[i];
    for (u32 j = 0; j < raw.predNum[i]; j++) {
      const u32 p = raw.predOff[i] + j; const u32 sc = raw.predCtr[p], sa = raw.predActor[p];
      succ[p] = (sc == NULL32 || sa == NULL32) ? 0 : pack_id(sc, actor(sa));
      if (sc != NULL32 && sc > mx) mx = sc;
    }
    if (mx > *maxOp) atomic_max(maxOp, mx);
    if (bad) raise(errWord, KE_ACTOR_INDEX, i);
  }
};
struct KeySlotInitKernel { KeySlot* s; HD void operator()(size_t i) const { s[i].hash = 0; s[i].rep = 0xffffffffu; s[i].rank = 0; } };
struct InsertFlagKernel { DocRows w; u32* flag; HD void operator()(size_t r) const { flag[r] = (w.keyStrLen[r] == NULL32 && (w.flags[r] & F_INSERT)) ? 1u : 0u; } };
struct GatherU32Kernel { const u32* src; const u32* idx; u32* out; HD void operator()(size_t i) const { out[i] = src[idx[i]]; } };
struct GatherToU64Kernel { const u32* src; const u32* idx; u64* out; HD void operator()(size_t i) const { out[i] = src[idx[i]]; } };
struct NewSuccFlagKernel { const u32* pairPos; const u32* pairTime; u32* newCnt; HD void operator()(size_t q) const { if (pairTime[q] != 0) atomic_add(&newCnt[pairPos[q]], 1u); } };
struct ObjPosKernel { const u32* perm; const u32* objRow; const u32* pos; u32* objPos; HD void operator()(size_t p) const { const u32 o = objRow[perm[p]]; objPos[p] = o == ROW_NONE ? ROW_NONE : pos[o]; } };
struct SuccCntFromOffKernel { const u32* off; u32* cnt; HD void operator()(size_t p) const { cnt[p] = off[p + 1] - off[p]; } };
struct EditKeyKernel { const u32* objKey; const EditRec* e; u64* key; u32* val; HD void operator()(size_t j) const { key[j] = objKey[j]; val[j] = (u32)j; } };
struct EditTimeKeyKernel { const u32* t; u64* key; u32* val; HD void operator()(size_t j) const { key[j] = t[j]; val[j] = (u32)j; } };
struct EditGatherKernel {   // permutes the parallel edit arrays (posIn / keyIn may be null)
  const EditRec* in; const u64* elemIn; const u32* posIn; const u32* keyIn; const u32* idx; EditRec* out; u64* elemOut; u32* posOut; u32* keyOut;
  HD void operator()(size_t j) const { const u32 s = idx[j]; out[j] = in[s]; elemOut[j] = elemIn[s]; if (posIn) posOut[j] = posIn[s]; if (keyIn) keyOut[j] = keyIn[s]; }
};
struct OffsetIotaKernel { u32* val; u32 base; HD void operator()(size_t j) const { val[j] = base + (u32)j; } };
struct EditTimeKeyAtKernel { const u32* t; u32 base; u64* key; u32* val; HD void operator()(size_t j) const { key[j] = t[base + j]; val[j] = base + (u32)j; } };

}  // namespace amg
