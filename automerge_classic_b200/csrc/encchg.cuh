// amgpu — kernels #10: encodeChange (reference columnar.js:710-739) over the changes of a change table (the layout
// amg_decode_changes returns, include/amgpu.h) into binary changes and their hashes.
//
// Only Engine::encodeChanges launches these. Per call (n changes of a table staged in device memory; the host has checked
// the header's sections):
//   EncChangeKernel     one thread per change: the record's ranges (ops, preds, actor entries, message, deps, extra bytes),
//                       seq / startOp / time, and the change's pred count                                  -> ops, preds, actors
//   (scans of ops, preds and actor entries per change)
//   EncOpKernel         one thread per op: decodeChange's op checks in encodeOps' order (object, key, action, value, child,
//                       preds), every offset the writer will read
//   actor ids           ranked over the call: LSD radix sort of the referenced entries (length, then 8-byte chunks from the
//                       last), equal neighbours share a rank
//   EncActorPairKernel  one thread per op: (change, actor rank) for every actor the op mentions; sorted and made unique by
//                       the history kernels (HistUniqueKernel, HistOtherFillKernel, HistLowerBoundKernel): the change's other
//                       actors in parseAllOpIds order (columnar.js:133-170)
//   EncPrepKernel       one thread per change: local actor numbers, delta values, preds sorted by (counter, actor id)
//   EncColSizeKernel    one thread per (column, change): the column's length (hist_column, history.cuh)
//   EncChangeHeadKernel one thread per change; pass 0: the container's length (write_change_head, history.cuh) -> 64-bit
//                       scan -> output offsets; pass 1: container header, body head, directory, extra bytes
//   EncColWriteKernel   one thread per (column, change): the column's bytes
//   EncHashKernel       one thread per change: deps sorted by hash bytes into place, SHA-256 (hist_sha256), checksum
// Errors: one error word per phase (raise(): smallest item wins); the change reported is the smallest failing change, and for
// it the error of its earliest phase.
#pragma once
#include "changes.cuh"
#include "history.cuh"

namespace amg {

static const u64 ENC_MAX_SAFE = (1ULL << 53) - 1;   // Number.MAX_SAFE_INTEGER: the encoder's LEB128 range (encoding.js)
enum EncErr { EE_CHG_OPS = 0xa0, EE_CHG_PREDS, EE_CHG_ACTORS, EE_ACTOR_ENTRY, EE_CHG_MSG, EE_CHG_DEPS, EE_CHG_EXTRA, EE_NUM_RANGE, EE_TOO_LARGE,
              EE_OP_KEYSTR, EE_OP_VALUE, EE_OP_PREDS, EE_OBJ, EE_KEY, EE_KEY_ACTOR, EE_ACTION, EE_CHLD_ACTOR, EE_CHLD_NULL, EE_PRED_ACTOR, EE_PRED_NULL,
              EE_CHANGE_SIZE };
// EP_SIZE: a change whose encoding may reach 4 GiB. Its own word, after the op checks: an op error of the same change wins.
enum EncPhase { EP_CHANGES = 0, EP_OPS, EP_SIZE, EP_NUM };
// The writer counts a change's bytes in 32 bits (ByteSink, column lengths, container length). Ops may share one value or key
// string, so the bytes a change writes are not bounded by the table's size: every change is bounded in 64 bits first. Per
// op: 9 numeric columns of at most 20 bytes a value (a LEB128 value and the header of its own literal run), the insert run,
// the key string (length, bytes, run header), the value bytes, and 40 bytes per pred (two numeric columns). Per change: the
// header, the actor table, the directory and the extra bytes.
static const u64 ENC_OP_BOUND = 9 * 20 + 10 + 10, ENC_PRED_BOUND = 40, ENC_CHANGE_BOUND = 64 + HC_NUM * 20, ENC_SIZE_LIMIT = 0xfff00000ULL;

// the staged table (sections checked by the host: inside the table, 8-byte aligned)
struct EncTable {
  const u8* t; u64 len; u64 nOps, nPreds, nActors; const ChangeRec* ch; const OpRec* ops; const u32* preds; const ActorRef* actors;
  // applyLocalChange: the author's previous change, hashes + 32 * *prevIdx, is one more dependency of every change of the
  // call; the deps are then the sorted union without repeats (backend.js:76-79). prevIdx == nullptr: no extra dependency.
  const u8* prevHashes = nullptr; const u32* prevIdx = nullptr;
  HD bool inside(u64 off, u64 n) const { return off <= len && n <= len - off; }
  HD const u8* dep(const ChangeRec& r, u32 i) const { return t + r.depsOff + 32ULL * i; }
  HD const u8* extraDep() const { return prevIdx ? prevHashes + 32ULL * *prevIdx : nullptr; }
};
HD bool enc_same_hash(const u8* a, const u8* b) { for (int k = 0; k < 32; k++) if (a[k] != b[k]) return false; return true; }
// the number of dependencies the header lists (the deps section is in range)
HD u32 enc_num_deps(const EncTable& T, const ChangeRec& r) {
  const u8* x = T.extraDep();
  if (!x) return r.nDeps;
  u32 n = 1;
  for (u32 i = 0; i < r.nDeps; i++) {
    bool seen = enc_same_hash(T.dep(r, i), x);
    for (u32 j = 0; j < i && !seen; j++) seen = enc_same_hash(T.dep(r, i), T.dep(r, j));
    if (!seen) n++;
  }
  return n;
}
HD bool enc_set_or_inc(u32 action) { return action == 1 || action == 5; }   // encodeValue writes a value for these only (columnar.js:260)
HD bool enc_map_key(const OpRec& o) { return o.keyStrLen != NULL32 && o.keyStrLen > 0; }
HD bool enc_elem_key(const OpRec& o) { return !enc_map_key(o) && o.keyCtr != NULL32 && o.keyCtr > 0; }
HD bool enc_has_child(const OpRec& o) { return o.chldCtr != NULL32 && o.chldCtr != 0; }   // columnar.js:404-410

// change records: ranges, numbers, the change's pred count. A failing change gets no ops, preds or actors.
struct EncChangeKernel {
  EncTable T; u32* nOps; u32* nPreds; u32* nActors; u32* maxActorLen; u64* err; u64* sizeErr;
  HD void fail(size_t c, u32 code) const { raise(err, code, c); nOps[c] = 0; nPreds[c] = 0; nActors[c] = 0; }
  HD void operator()(size_t c) const {
    nOps[c] = 0; nPreds[c] = 0; nActors[c] = 0;
    const ChangeRec& r = T.ch[c];
    if (r.firstOp > T.nOps || r.nOps > T.nOps - r.firstOp) { fail(c, EE_CHG_OPS); return; }
    if (r.firstPred > T.nPreds || r.nPreds > T.nPreds - r.firstPred) { fail(c, EE_CHG_PREDS); return; }
    if (r.nActors == 0 || r.actorFirst > T.nActors || r.nActors > T.nActors - r.actorFirst) { fail(c, EE_CHG_ACTORS); return; }
    u32 maxLen = 0; u64 bound = ENC_CHANGE_BOUND;
    for (u32 a = 0; a < r.nActors; a++) {
      const ActorRef e = T.actors[r.actorFirst + a];
      if (!T.inside(e.off, e.len)) { fail(c, EE_ACTOR_ENTRY); return; }
      if (e.len > maxLen) maxLen = e.len;
      bound += 10 + (u64)e.len;
    }
    if (!T.inside(r.msgOff, r.msgLen)) { fail(c, EE_CHG_MSG); return; }
    if (!T.inside(r.depsOff, 32ULL * r.nDeps)) { fail(c, EE_CHG_DEPS); return; }
    if (r.hasExtra && !T.inside(r.extraOff, r.extraLen)) { fail(c, EE_CHG_EXTRA); return; }
    if (r.seq > ENC_MAX_SAFE || r.startOp > ENC_MAX_SAFE || r.time > (long long)ENC_MAX_SAFE || r.time < -(long long)ENC_MAX_SAFE) { fail(c, EE_NUM_RANGE); return; }
    u64 preds = 0;
    bound += 10 + (u64)r.msgLen + 32ULL * ((u64)r.nDeps + (T.prevIdx ? 1 : 0)) + (r.hasExtra ? (u64)r.extraLen : 0);
    for (u64 i = 0; i < r.nOps; i++) {   // (fields the op checks have not seen yet only make the bound larger)
      const OpRec& o = T.ops[r.firstOp + i];
      preds += o.predNum;
      bound += ENC_OP_BOUND + ENC_PRED_BOUND * o.predNum + (enc_map_key(o) ? (u64)o.keyStrLen : 0) + (enc_set_or_inc(o.action) && o.valLen != NULL32 ? (u64)(o.valLen >> 4) : 0);
    }
    if (preds > 0x7fffffffULL) { fail(c, EE_TOO_LARGE); return; }
    if (bound >= ENC_SIZE_LIMIT) raise(sizeErr, EE_CHANGE_SIZE, c);   // (ops still checked: their errors come first)
    nOps[c] = (u32)r.nOps; nPreds[c] = (u32)preds; nActors[c] = r.nActors;
    atomic_max(maxActorLen, maxLen);
  }
};

// change of op j (j in [0, total ops)): the last c with opBase[c] <= j (changes without ops share a base with the next)
HD size_t enc_change_of(const u32* opBase, size_t n, u64 j) {
  size_t lo = 0, hi = n;
  while (hi - lo > 1) { const size_t mid = (lo + hi) / 2; if (opBase[mid] <= j) lo = mid; else hi = mid; }
  while (lo + 1 < n && opBase[lo + 1] <= j) lo++;
  return lo;
}

// the op checks, in encodeOps' order (columnar.js:370-436) with decodeChange's actor check (columnar.js:488) and decodeValue
// (columnar.js:300-329) on every value written; slot count for the actor pairs
struct EncOpKernel {
  EncTable T; const u32* opBase; size_t n; u32* slotCnt; u64* err;
  HD void operator()(size_t j) const {
    const size_t c = enc_change_of(opBase, n, j); const ChangeRec& r = T.ch[c];
    const OpRec& o = T.ops[r.firstOp + (j - opBase[c])]; const u32 na = r.nActors;
    slotCnt[j] = 0;
    if (o.objCtr != NULL32 && (o.objCtr == 0 || o.objActor >= na)) { raise(err, EE_OBJ, j); return; }
    if (enc_map_key(o)) { if (!T.inside(o.keyStrOff, o.keyStrLen)) { raise(err, EE_OP_KEYSTR, j); return; } }
    else if (enc_elem_key(o)) { if (o.keyActor >= na) { raise(err, o.keyActor == NULL32 ? EE_KEY : EE_KEY_ACTOR, j); return; } }
    else if (!(o.keyCtr == 0 && o.insert)) { raise(err, EE_KEY, j); return; }
    if (o.action == NULL32) { raise(err, EE_ACTION, j); return; }
    if (enc_set_or_inc(o.action) && o.valLen != NULL32) {
      if (!T.inside(o.valOff, o.valLen >> 4)) { raise(err, EE_OP_VALUE, j); return; }
      if (o.valLen > 2) { if (const u32 e = decode_value_error(T.t, o.valLen, o.valOff)) { raise(err, e, j); return; } }
    }
    if (enc_has_child(o) && o.chldActor >= na) { raise(err, o.chldActor == NULL32 ? EE_CHLD_NULL : EE_CHLD_ACTOR, j); return; }
    if (o.predFirst > T.nPreds || o.predNum > T.nPreds - o.predFirst) { raise(err, EE_OP_PREDS, j); return; }
    for (u32 k = 0; k < o.predNum; k++) {
      const u32 a = T.preds[2 * ((u64)o.predFirst + k)], ctr = T.preds[2 * ((u64)o.predFirst + k) + 1];
      if (ctr == NULL32) { raise(err, EE_PRED_NULL, j); return; }
      if (a >= na) { raise(err, EE_PRED_ACTOR, j); return; }
    }
    slotCnt[j] = 3 + o.predNum;
  }
};

// ---------------------------------------------------------------- actor ids ranked over the call
// (The op set's key ranking, opset.cuh, is not reused: it interns keys by hash from DocRows and orders them by their UTF-16
// form, as JavaScript compares strings. Actor ids order by their bytes, which is their hex text order, so a plain LSD radix
// sort over 8-byte chunks with radix_sort_pairs ranks them.)
// entries [actorBase[c], actorBase[c] + nActors[c]) are change c's actor table
struct EncActorListKernel {
  EncTable T; const u32* nActors; const u32* actorBase; u32* entOff; u32* entLen;
  HD void operator()(size_t c) const { const ChangeRec& r = T.ch[c]; for (u32 a = 0; a < nActors[c]; a++) { const ActorRef e = T.actors[r.actorFirst + a]; entOff[actorBase[c] + a] = e.off; entLen[actorBase[c] + a] = e.len; } }
};
// sort key of the entry at sorted position i: chunk < 0 its length, else id bytes [8 chunk, 8 chunk + 8) big endian, zero padded
struct EncActorKeyKernel {
  const u8* t; const u32* entOff; const u32* entLen; const u32* order; int chunk; u64* key; u32* val;
  HD void operator()(size_t i) const {
    const u32 e = order ? order[i] : (u32)i;
    if (!order) val[i] = e;
    if (chunk < 0) { key[i] = entLen[e]; return; }
    u64 k = 0; const u32 at = 8 * (u32)chunk, len = entLen[e];
    for (u32 b = 0; b < 8; b++) k = (k << 8) | (at + b < len ? t[entOff[e] + at + b] : 0u);
    key[i] = k;
  }
};
HD bool enc_same_id(const u8* t, const u32* entOff, const u32* entLen, u32 a, u32 b) {
  if (entLen[a] != entLen[b]) return false;
  for (u32 k = 0; k < entLen[a]; k++) if (t[entOff[a] + k] != t[entOff[b] + k]) return false;
  return true;
}
struct EncActorHeadKernel { const u8* t; const u32* entOff; const u32* entLen; const u32* order; u32* head; HD void operator()(size_t i) const { head[i] = (i == 0 || !enc_same_id(t, entOff, entLen, order[i], order[i - 1])) ? 1u : 0u; } };
// rank of every entry (hex string order = byte order, a prefix first); rep[rank] = one entry with that id
struct EncActorRankKernel {
  const u32* order; const u32* head; const u32* headScan; u32* entRank; u32* rep;
  HD void operator()(size_t i) const { const u32 rk = headScan[i] + head[i] - 1; entRank[order[i]] = rk; if (head[i]) rep[rk] = order[i]; }
};

// (change << 32 | rank) for the actors op j mentions (object, element key, child, preds), ~0 for none and for the author
struct EncActorPairKernel {
  EncTable T; const u32* opBase; size_t n; const u32* actorBase; const u32* entRank; const u32* slotBase; u64* key;
  HD void operator()(size_t j) const {
    const size_t c = enc_change_of(opBase, n, j); const ChangeRec& r = T.ch[c];
    const OpRec& o = T.ops[r.firstOp + (j - opBase[c])];
    const u32* rank = entRank + actorBase[c]; const u32 author = rank[0];
    auto mk = [&](u32 a) -> u64 { return rank[a] == author ? ~0ULL : (((u64)c << 32) | rank[a]); };
    u32 s = slotBase[j];
    key[s++] = o.objCtr != NULL32 ? mk(o.objActor) : ~0ULL;
    key[s++] = enc_elem_key(o) ? mk(o.keyActor) : ~0ULL;
    key[s++] = o.chldCtr != NULL32 && o.chldActor < r.nActors ? mk(o.chldActor) : ~0ULL;   // (parseAllOpIds counts a child of counter 0 too)
    for (u32 k = 0; k < o.predNum; k++) key[s++] = mk(T.preds[2 * ((u64)o.predFirst + k)]);
  }
};

// local actor number of an actor of rank `rk` in change c: author 0, others 1 + position in the change's sorted list
HD u32 enc_local_actor(const u64* other, const u32* otherStart, size_t c, u32 author, u32 rk) {
  if (rk == author) return 0;
  const u64 want = ((u64)c << 32) | rk;
  u32 lo = otherStart[c], hi = otherStart[c + 1];
  while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (other[mid] < want) lo = mid + 1; else hi = mid; }
  return 1 + (lo - otherStart[c]);
}
// per change: local actor numbers and delta values of its ops (in table order) and of its preds (sorted per op by counter,
// then actor id: columnar.js:423)
struct EncPrepKernel {
  EncTable T; const u32* opBase; const u32* predBase; const u32* actorBase; const u32* entRank; const u64* other; const u32* otherStart;
  u32* objA; u32* keyA; long long* keyDelta; u32* chA; long long* chDelta; u64* predKey; u32* predA; long long* predDelta;
  HD void operator()(size_t c) const {
    const ChangeRec& r = T.ch[c]; const u32 nOps = opBase[c + 1] - opBase[c];
    const u32* rank = entRank + actorBase[c]; const u32 author = rank[0];
    long long keyAbs = 0, chAbs = 0, predAbs = 0; u32 q = predBase[c];
    for (u32 i = 0; i < nOps; i++) {
      const OpRec& o = T.ops[r.firstOp + i]; const u32 j = opBase[c] + i;
      objA[j] = o.objCtr != NULL32 ? enc_local_actor(other, otherStart, c, author, rank[o.objActor]) : NULL32;
      if (enc_map_key(o)) { keyA[j] = NULL32; keyDelta[j] = NULLV; }
      else {
        const bool elem = enc_elem_key(o);   // else _head: actor null, counter 0 (columnar.js:190-193)
        keyA[j] = elem ? enc_local_actor(other, otherStart, c, author, rank[o.keyActor]) : NULL32;
        const long long abs = elem ? (long long)o.keyCtr : 0; keyDelta[j] = abs - keyAbs; keyAbs = abs;
      }
      if (enc_has_child(o)) { chA[j] = enc_local_actor(other, otherStart, c, author, rank[o.chldActor]); chDelta[j] = (long long)o.chldCtr - chAbs; chAbs = o.chldCtr; }
      else { chA[j] = NULL32; chDelta[j] = NULLV; }
      for (u32 k = 0; k < o.predNum; k++) {   // insertion sort by (counter, actor rank): pred lists are short
        const u64 p = 2 * ((u64)o.predFirst + k);
        const u64 key = ((u64)T.preds[p + 1] << 32) | rank[T.preds[p]];
        u32 at = q + k; while (at > q && predKey[at - 1] > key) { predKey[at] = predKey[at - 1]; at--; }
        predKey[at] = key;
      }
      for (u32 k = 0; k < o.predNum; k++, q++) {
        predA[q] = enc_local_actor(other, otherStart, c, author, (u32)(predKey[q] & 0xffffffffu));
        const long long abs = (long long)(predKey[q] >> 32); predDelta[q] = abs - predAbs; predAbs = abs;
      }
    }
  }
};

// op source of the column writer over one change of the table
struct EncChangeSrc {
  u32 nOps, nPreds; const u8* t; const OpRec* ops /* the change's first op */; u32 j0, q0;
  const u32* objA; const u32* keyA; const long long* keyDelta; const u32* chA; const long long* chDelta; const u32* predA; const long long* predDelta;
  HD u32 valLen(const OpRec& o) const { return enc_set_or_inc(o.action) && o.valLen != NULL32 ? o.valLen : 0u; }   // encodeValue: null for other actions
  HD bool num(int col, u32 i, long long& x) const {
    const OpRec& o = ops[i]; const u32 j = j0 + i;
    auto u = [&](u32 v) { if (v == NULL32) return false; x = v; return true; };
    auto d = [&](long long v) { if (v == NULLV) return false; x = v; return true; };
    switch (col) {
      case HC_OBJ_ACTOR: return u(objA[j]);
      case HC_OBJ_CTR: return u(o.objCtr);
      case HC_KEY_ACTOR: return u(keyA[j]);
      case HC_KEY_CTR: return d(keyDelta[j]);
      case HC_ACTION: x = o.action; return true;
      case HC_VAL_LEN: x = valLen(o); return true;
      case HC_CHLD_ACTOR: return u(chA[j]);
      case HC_CHLD_CTR: return d(chDelta[j]);
      case HC_PRED_NUM: x = o.predNum; return true;
      case HC_PRED_ACTOR: x = predA[q0 + i]; return true;
      case HC_PRED_CTR: x = predDelta[q0 + i]; return true;
      default: return false;
    }
  }
  HD bool keyNull(u32 i) const { return !enc_map_key(ops[i]); }
  HD bool keySame(u32 a, u32 b) const {
    const OpRec& x = ops[a]; const OpRec& y = ops[b]; if (x.keyStrLen != y.keyStrLen) return false;
    for (u32 k = 0; k < x.keyStrLen; k++) if (t[x.keyStrOff + k] != t[y.keyStrOff + k]) return false;
    return true;
  }
  HD void keyPut(ByteSink& out, u32 i) const { out.uleb(ops[i].keyStrLen); out.bytes(t + ops[i].keyStrOff, ops[i].keyStrLen); }
  HD bool insert(u32 i) const { return ops[i].insert != 0; }
  HD void valRaw(ByteSink& out, u32 i) const { const OpRec& o = ops[i]; out.bytes(t + o.valOff, valLen(o) >> 4); }
};
struct EncCols {   // everything EncChangeSrc reads besides the table
  const u32* opBase; const u32* predBase; const u32* objA; const u32* keyA; const long long* keyDelta; const u32* chA; const long long* chDelta; const u32* predA; const long long* predDelta;
  HD EncChangeSrc src(const EncTable& T, size_t c) const {
    return EncChangeSrc{opBase[c + 1] - opBase[c], predBase[c + 1] - predBase[c], T.t, T.ops + T.ch[c].firstOp, opBase[c], predBase[c], objA, keyA, keyDelta, chA, chDelta, predA, predDelta};
  }
};
struct EncOthers {   // the other actors of change c: ids by rank (other: (c << 32 | rank), sorted)
  const u64* other; u32 count; const u32* rep; const u32* entOff; const u32* entLen; const u8* t;
  HD u32 n() const { return count; }
  HD void put(ByteSink& b, u32 q) const { const u32 e = rep[(u32)(other[q] & 0xffffffffu)]; b.uleb(entLen[e]); b.bytes(t + entOff[e], entLen[e]); }
};

// column lengths: colLen[col * n + c]
struct EncColSizeKernel {
  EncTable T; EncCols cols; size_t n; u32* colLen;
  HD void operator()(size_t i) const { const int col = (int)(i / n); const size_t c = i % n; ByteSink s{nullptr, 0}; hist_column(s, cols.src(T, c), col); colLen[i] = s.n; }
};
// pass 0: container length of change c; pass 1: its header, body head and directory, and the extra bytes behind the columns
struct EncChangeHeadKernel {
  int pass; EncTable T; size_t n; const u32* colLen; const u32* actorBase; const u32* entOff; const u32* entLen; const u32* rep; const u64* other; const u32* otherStart;
  u32* outLen; const u64* outOff; u8* out; u64* dataAt; u64* depsAt; u64* bodyAt;
  HD void operator()(size_t c) const {
    const ChangeRec& r = T.ch[c]; u32 len[HC_NUM]; u32 dataLen = 0;
    for (int col = 0; col < HC_NUM; col++) { len[col] = colLen[(size_t)col * n + c]; dataLen += len[col]; }
    const u32 a0 = actorBase[c];
    const ChangeHead h{enc_num_deps(T, r), T.t + entOff[a0], entLen[a0], r.seq, r.startOp, r.time, T.t + r.msgOff, r.msgLen};
    const EncOthers others{other + otherStart[c], otherStart[c + 1] - otherStart[c], rep, entOff, entLen, T.t};
    const u32 extra = r.hasExtra ? r.extraLen : 0;
    ByteSink w{pass ? out + outOff[c] : nullptr, 0};
    u32 dAt = 0, bAt = 0, cAt = 0;
    const u32 total = write_change_head(w, h, others, len, extra, &dAt, &bAt, &cAt);
    if (pass == 0) { outLen[c] = total; return; }
    dataAt[c] = outOff[c] + cAt; depsAt[c] = outOff[c] + dAt; bodyAt[c] = outOff[c] + bAt;
    w.n = cAt + dataLen; w.bytes(T.t + r.extraOff, extra);
  }
};
struct EncColWriteKernel {
  EncTable T; EncCols cols; size_t n; const u32* colLen; const u64* dataAt; u8* out;
  HD void operator()(size_t i) const {
    const int col = (int)(i / n); const size_t c = i % n;
    if (!colLen[i]) return;
    u64 at = dataAt[c]; for (int k = 0; k < col; k++) at += colLen[(size_t)k * n + c];
    ByteSink w{out + at, 0}; hist_column(w, cols.src(T, c), col);
  }
};
// dependency hashes (given as bytes: no level-by-level walk) sorted into place, then the change's hash and checksum
struct EncHashKernel {
  EncTable T; const u64* outOff; const u32* outLen; const u64* depsAt; const u64* bodyAt; u8* out; u8* hashes;
  HD void operator()(size_t c) const {
    const ChangeRec& r = T.ch[c]; u8* dst = out + depsAt[c]; const u8* x = T.extraDep(); u32 n = 0;
    auto put = [&](const u8* h) {   // insertion sort by hash bytes (columnar.js:717; deps are few); with x, repeats are dropped
      if (x) for (u32 k = 0; k < n; k++) if (enc_same_hash(dst + 32 * k, h)) return;
      u32 pos = n++;
      while (pos > 0) { const u8* prev = dst + 32 * (pos - 1); int cmp = 0; for (int b = 0; b < 32 && !cmp; b++) cmp = (int)prev[b] - (int)h[b]; if (cmp <= 0) break; for (int b = 0; b < 32; b++) dst[32 * pos + b] = prev[b]; pos--; }
      for (int b = 0; b < 32; b++) dst[32 * pos + b] = h[b];
    };
    for (u32 i = 0; i < r.nDeps; i++) put(T.dep(r, i));
    if (x) put(x);
    u8 digest[32]; hist_sha256(out + bodyAt[c], (u32)(outOff[c] + outLen[c] - bodyAt[c]), digest);
    for (int b = 0; b < 32; b++) hashes[c * 32 + b] = digest[b];
    for (int b = 0; b < 4; b++) out[outOff[c] + 4 + b] = digest[b];
  }
};
struct EncOutLen64 { const u32* len; HD u64 operator()(size_t i) const { return len[i]; } };

}  // namespace amg
