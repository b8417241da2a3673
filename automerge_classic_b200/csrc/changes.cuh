// amgpu — kernels #9: decodeChange / decodeChanges (reference columnar.js:770-776, 843-857) into one flat change table.
//
// Only Engine::decodeChanges launches these; the apply path keeps its own kernels. Per call (n changes, bytes in one device
// arena, DEFLATEd ones already inflated behind them):
//   ChgContainerKernel  one thread per change: split_container's reads (magic, chunk type, length, body)  -> container length
//   ShaKernel           (decode.cuh) SHA-256 of [8, container end): the hash and the checksum check
//   ChgHeaderKernel     one thread per change: trailing data, chunk type, decodeChangeHeader, column directory, every known
//                       column validated in the reference's order and counted; op count = the longest column (columnar.js:580)
//   (scans of ops, preds, actors and bytes per change)
//   ChgColumnsKernel    one thread per (column, change): decode_one_column_t (decode.cuh) for the op columns, plus the child
//                       columns chldActor / chldCtr (0x61 / 0x63), which the apply path does not read
//   ChgRecordKernel     one thread per change: change record and its actor table entries
//   ChgBytesKernel      one thread per 64 output bytes: the change containers gathered into the table's bytes section
//   ChgOpKernel         one thread per op: op record, pred records, and decodeChange's op checks (actor indexes, child
//                       columns, decodeValue of every value, pred order)
// Errors: each phase has its own error word (raise(): smallest item wins). The change reported is the smallest failing
// change over all phases, and for that change the error of its earliest phase: what the sequential reference meets first.
#pragma once
#include "decode.cuh"

namespace amg {

static const u64 CHG_MAGIC = 0x31474843474d41ULL;   // "AMGCHG1"
enum { CHG_HDR_WORDS = 12 };
// error codes of decodeChange's own checks (the KErr codes of decode.cuh keep their meaning)
enum DecErr { DE_CHUNK_TYPE_N = 0x80 /* Unexpected chunk type: N */, DE_OBJ_ACTOR, DE_KEY_ACTOR, DE_CHLD_ACTOR, DE_PRED_ACTOR, DE_CHLD_MISMATCH,
              DE_PRED_ORDER, DE_PRED_NULL /* a null pred id that would have to be ordered: the host mirror cannot compare it */ };
enum DecPhase { DP_INFLATE = 0, DP_CONTAINER, DP_SHA, DP_HEADER, DP_COLUMNS, DP_OPS, DP_NUM };
static const int CHG_COLS = 16;   // column slots per change: the NCOLS known columns (ColIx), then unused

struct alignas(8) ChangeRec {   // 128 bytes (layout: include/amgpu.h)
  u8 hash[32]; u64 seq, startOp; long long time;
  u32 msgOff, msgLen, depsOff, nDeps, actorFirst, nActors, extraOff, extraLen, hasExtra, pad;
  u64 firstOp, nOps, firstPred, nPreds;
};
struct OpRec {   // 64 bytes; NULL32 = null
  u32 objActor, objCtr, keyActor, keyCtr, keyStrOff, keyStrLen, insert, action, valLen, valOff, chldActor, chldCtr, predFirst, predNum, change, pad;
};
struct ActorRef { u32 off, len; };

// split_container (columnar.js:688-708 decodeContainerHeader): magic, checksum, chunk type, LEB128 length, body
struct ChgContainerKernel {
  const u8* arena; const u32* chOff; const u32* chLen; u32* cLen; u64* err;
  HD void operator()(size_t c) const {
    const u32 off = chOff[c], len = chLen[c]; cLen[c] = 0;
    const u8* p = arena + off;
    if (len < 4) { raise(err, KE_SUBARRAY, c); return; }
    if (p[0] != 0x85 || p[1] != 0x6f || p[2] != 0x4a || p[3] != 0x83) { raise(err, KE_MAGIC, c); return; }
    if (len < 9) { raise(err, KE_SUBARRAY, c); return; }
    ByteReader r(arena, off + 9, off + len);
    const u64 l = r.uleb(); if (r.err) { raise(err, r.err, c); return; }
    r.skip(l); if (r.err) { raise(err, r.err, c); return; }
    cLen[c] = r.pos - off;
  }
};

// counts of one column the way the host mirror decodes it (rle_decode / delta_decode / bool_decode): every record is read
template <class S> HD u32 chg_column_count(const S& src, u32 id, u32 off, u32 end, u32* err) {
  if (id == 0x34) {   // BooleanDecoder: runs of alternating values, a zero-length run only first
    ByteReaderT<S> r(src, off, end); u64 n = 0; bool first = true; *err = 0;
    while (!r.done()) {
      const u64 k = r.uleb(); if (r.err) { *err = r.err; return 0; }
      if (k == 0 && !first) { *err = KE_BOOL_ZERO; return 0; }
      first = false; n += k;
      if (n > 0xfffffffeULL) { *err = KE_TOO_LARGE; return 0; }
    }
    return (u32)n;
  }
  return rle_count_values_t(src, off, end, err, (id & 7) == 3 ? 1 : (id & 7) == 5 ? 2 : 0);
}

// decodeChange's container checks after the hash, decodeChangeHeader (columnar.js:635-652), decodeColumnInfo (:609-624),
// the column split (:741-765) and decodeColumns' row count (:577-607). On failure the change gets no ops, preds, actors or bytes.
struct ChgHeaderKernel {
  const u8* arena; const u32* chOff; const u32* chLen; const u32* cLen; const u8* hashes; ChangeMeta* meta; u32* colOff /* [CHG_COLS][n] */; u32* colLen;
  u32* nOps; u32* nPreds; u32* nActors; u32* nBytes; size_t n; u64* err;
  HD void fail(size_t c, u32 code) const { raise(err, code, c); nOps[c] = 0; nPreds[c] = 0; nActors[c] = 0; nBytes[c] = 0; }
  HD void operator()(size_t c) const {
    nOps[c] = 0; nPreds[c] = 0; nActors[c] = 0; nBytes[c] = 0;
    for (int k = 0; k < CHG_COLS; k++) { colOff[(size_t)k * n + c] = 0; colLen[(size_t)k * n + c] = 0; }
    const u32 off = chOff[c], len = chLen[c], cl = cLen[c];
    if (cl == 0) return;   // the container phase failed
    const u8* p = arena + off; const u8* h = hashes + c * 32;
    if (h[0] != p[4] || h[1] != p[5] || h[2] != p[6] || h[3] != p[7]) return;   // the SHA phase reported it
    if (cl != len) { fail(c, KE_TRAILING); return; }
    if (p[8] != 1) { fail(c, DE_CHUNK_TYPE_N); return; }
    ByteReader r(arena, off + 9, off + len); r.uleb();
    ChangeMeta m; memset(&m, 0, sizeof(m)); m.off = off; m.len = len;
#define CHG_CHECK() do { if (r.err) { fail(c, r.err); return; } } while (0)
    const u64 nDeps = r.uleb(); CHG_CHECK();
    m.depsOff = r.pos;
    for (u64 i = 0; i < nDeps; i++) { r.skip(32); CHG_CHECK(); }
    m.nDeps = (u32)nDeps;
    const u64 actorLen = r.uleb(); CHG_CHECK(); m.actorOff = r.pos; m.actorLen = (u32)actorLen; r.skip(actorLen); CHG_CHECK();
    m.seq = r.uleb(); CHG_CHECK(); m.startOp = r.uleb(); CHG_CHECK(); m.time = r.sleb(); CHG_CHECK();
    const u64 msgLen = r.uleb(); CHG_CHECK(); m.msgOff = r.pos; m.msgLen = (u32)msgLen; r.skip(msgLen); CHG_CHECK();
    const u64 nOther = r.uleb(); CHG_CHECK(); m.otherOff = r.pos;
    for (u64 i = 0; i < nOther; i++) { const u64 l = r.uleb(); CHG_CHECK(); r.skip(l); CHG_CHECK(); }
    if (nOther > 0xfffffff0ULL) { fail(c, KE_TOO_LARGE); return; }
    m.nOther = (u32)nOther;
    const u64 nCols = r.uleb(); CHG_CHECK();
    m.dirOff = r.pos; long long lastId = -1;
    for (u64 i = 0; i < nCols; i++) {
      const u64 id = r.uleb(); CHG_CHECK(); r.uleb(); CHG_CHECK();
      if (lastId >= 0 && (id & ~8ULL) <= ((u64)lastId & ~8ULL)) { fail(c, KE_COL_ORDER); return; }
      lastId = (long long)id;
    }
    m.dataOff = r.pos;
    ByteReader d(arena, m.dirOff, m.dataOff);
    for (u64 i = 0; i < nCols; i++) {
      const u64 id = d.uleb(), l = d.uleb();
      if (id & 8) { fail(c, KE_COL_DEFLATE); return; }
      const u32 at = r.pos; r.skip(l); CHG_CHECK();
      const int ix = id < 0x80 ? col_index_of((u32)id) : -1;
      if (ix >= 0) { colOff[(size_t)ix * n + c] = at; colLen[(size_t)ix * n + c] = (u32)l; }
    }
#undef CHG_CHECK
    m.extraOff = r.pos; m.extraLen = off + len - r.pos;
    // decodeChange reads the action column first, then the other op columns in directory order, then the pred actor
    // and counter columns; the row count is the longest of the op columns
    const u32 order[13] = {0x42, 0x01, 0x02, 0x11, 0x13, 0x15, 0x34, 0x56, 0x61, 0x63, 0x70, 0x71, 0x73};
    u32 rows = 0;
    for (int k = 0; k < 13; k++) {
      const int ix = col_index_of(order[k]); const u32 co = colOff[(size_t)ix * n + c], cn = colLen[(size_t)ix * n + c];
      u32 e = 0; const u32 cnt = chg_column_count(PtrSrc{arena}, order[k], co, co + cn, &e);
      if (e) { fail(c, e); return; }
      if (order[k] != 0x71 && order[k] != 0x73 && cnt > rows) rows = cnt;
    }
    u32 e = 0; const int pn = CX_PRED_NUM;
    const u64 preds = rle_sum_values(arena, colOff[(size_t)pn * n + c], colOff[(size_t)pn * n + c] + colLen[(size_t)pn * n + c], rows, &e);
    if (e) { fail(c, e); return; }
    if (preds > 0x7fffffffULL || (u64)rows + preds > 0x7fffffffULL) { fail(c, KE_TOO_LARGE); return; }
    m.nOps = rows; m.nPreds = (u32)preds; meta[c] = m;
    nOps[c] = rows; nPreds[c] = (u32)preds; nActors[c] = 1 + m.nOther; nBytes[c] = len;
  }
};

// 64-bit totals of ops, preds and actor table entries over the call (the per-change counts are scanned in 32 bits: the
// host refuses a call whose totals do not fit before anything is sized by the scans). Every lane reaches the reduction.
HD void chg_warp_add64(u64* target, u32 v) {
#if defined(__CUDA_ARCH__)
  const unsigned active = __activemask();
  const u32 hi = __reduce_add_sync(active, v >> 16), lo = __reduce_add_sync(active, v & 0xffffu);   // each < 2^21: no wrap
  if ((int)(threadIdx.x & 31) == __ffs(active) - 1) atomicAdd(reinterpret_cast<unsigned long long*>(target), ((unsigned long long)hi << 16) + lo);
#else
  *target += v;
#endif
}
struct ChgTotalsKernel {
  const u32* nOps; const u32* nPreds; const u32* nActors; u64* totals;
  HD void operator()(size_t c) const { chg_warp_add64(totals, nOps[c]); chg_warp_add64(totals + 1, nPreds[c]); chg_warp_add64(totals + 2, nActors[c]); }
};

// The op columns of one change into SoA rows (decode_one_column_t), and the child columns. The columns were validated in
// full by ChgHeaderKernel; what is left to report is a value beyond the table's 32-bit fields.
struct ChgColumnsKernel {
  const u8* arena; const u32* colOff; const u32* colLen; const u32* nOps; const u32* nPreds; const u32* opBase; const u32* predBase; size_t n;
  RawRows rows; u32* chldActor; u32* chldCtr; u64* err;
  HD void operator()(size_t i) const {
    const int col = (int)(i / n); const size_t c = i % n;
    const u32 m = nOps[c]; if (m == 0 && (col != CX_PRED_ACTOR && col != CX_PRED_CTR)) return;
    const u32 co = colOff[(size_t)col * n + c], ce = co + colLen[(size_t)col * n + c], base = opBase[c], pb = predBase[c], np = nPreds[c];
    u32 kerr = 0;
    if (col == CX_VAL_RAW) return;
    if (col == CX_CHLD_ACTOR || col == CX_CHLD_CTR) {
      RleReader r(arena, co, ce, col == CX_CHLD_CTR ? 1 : 0); long long acc = 0;
      for (u32 k = 0; k < m; k++) {
        long long v = 0; u32 o, l; const bool nn = r.next(v, o, l);
        if (col == CX_CHLD_CTR) { if (nn) { acc += v; if (acc < 0 || acc > 0xfffffffeLL) kerr = KE_TOO_LARGE; } chldCtr[base + k] = nn ? (u32)acc : NULL32; }
        else { if (nn && (u64)v > 0xfffffffeULL) kerr = KE_TOO_LARGE; chldActor[base + k] = nn ? (u32)v : NULL32; }
      }
    } else {
      const int vr = CX_VAL_RAW;
      kerr = decode_one_column_t(PtrSrc{arena}, col, m, base, co, ce, colOff[(size_t)vr * n + c], colLen[(size_t)vr * n + c], pb, np, rows);
      if (col == CX_VAL_LEN && kerr == KE_SUBARRAY) kerr = 0;   // values past the raw column: reported per op, in op order (ChgOpKernel)
    }
    if (kerr) raise(err, kerr, c);
  }
};

// change record + actor table entries (offsets into the table: bytesOff + the change's place in the bytes section)
struct ChgRecordKernel {
  const u8* arena; const ChangeMeta* meta; const u8* hashes; const u32* nOps; const u32* nActors; const u32* opBase; const u32* predBase; const u32* actorBase;
  const u32* byteBase; u64 bytesOff; ChangeRec* recs; ActorRef* actors;
  HD void operator()(size_t c) const {
    ChangeRec rec; memset(&rec, 0, sizeof(rec));
    for (int k = 0; k < 32; k++) rec.hash[k] = hashes[c * 32 + k];
    const u32 na = nActors[c];
    if (na > 0) {   // (a change that failed has no actors: its record stays empty)
      const ChangeMeta& m = meta[c]; const u32 shift = (u32)(bytesOff + byteBase[c]) - m.off;
      rec.seq = m.seq; rec.startOp = m.startOp; rec.time = m.time;
      rec.msgOff = m.msgOff + shift; rec.msgLen = m.msgLen; rec.depsOff = m.depsOff + shift; rec.nDeps = m.nDeps;
      rec.extraOff = m.extraOff + shift; rec.extraLen = m.extraLen; rec.hasExtra = m.extraLen > 0;
      ActorRef* a = actors + actorBase[c]; a[0] = ActorRef{m.actorOff + shift, m.actorLen};
      ByteReader r(arena, m.otherOff, m.dirOff);
      for (u32 k = 1; k < na; k++) { const u32 l = (u32)r.uleb(); a[k] = ActorRef{r.pos + shift, l}; r.skip(l); }
    }
    rec.actorFirst = actorBase[c]; rec.nActors = na;
    rec.firstOp = opBase[c]; rec.nOps = nOps[c]; rec.firstPred = predBase[c]; rec.nPreds = predBase[c + 1] - predBase[c];
    recs[c] = rec;
  }
};

// the containers of the decoded changes, back to back: output bytes [64 i, 64 i + 64) of the section
struct ChgBytesKernel {
  const u8* arena; const u32* chOff; const u32* byteBase; size_t n; u32 total; u8* out;
  HD void operator()(size_t i) const {
    u32 at = (u32)(i * 64); const u32 end = at + 64 < total ? at + 64 : total;
    size_t lo = 0, hi = n;   // last change whose range starts at or before `at`
    while (hi - lo > 1) { const size_t mid = (lo + hi) / 2; if (byteBase[mid] <= at) lo = mid; else hi = mid; }
    size_t c = lo;
    while (at < end) {
      while (c + 1 < n && byteBase[c + 1] <= at) c++;
      const u32 stop = byteBase[c + 1] < end ? byteBase[c + 1] : end;
      const u8* src = arena + chOff[c] + (at - byteBase[c]);
      for (u32 k = 0; at + k < stop; k++) out[at + k] = src[k];
      at = stop;
    }
  }
};

// actor ids compared as the reference's hex text: bytewise, a prefix first
HD int chg_actor_cmp(const u8* tab, const ActorRef& a, const ActorRef& b) {
  const u32 l = a.len < b.len ? a.len : b.len;
  for (u32 k = 0; k < l; k++) if (tab[a.off + k] != tab[b.off + k]) return tab[a.off + k] < tab[b.off + k] ? -1 : 1;
  return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
}

// decodeOps (columnar.js:483-523) and the checks it makes, for op g of the call (errors keyed by g: the first failing op
// of the first failing change wins)
struct ChgOpKernel {
  const u8* arena; const u32* chOff; const u32* opBase; size_t n; RawRows rows; const u32* chldActor; const u32* chldCtr;
  const u32* colOff; const u32* colLen; const u32* nActors; const u32* actorBase; const u32* byteBase; u64 bytesOff;
  const u8* table /* the output buffer: actor ids are compared in its bytes section */; const ActorRef* actors; OpRec* ops; u32* preds; u64* err;
  HD void operator()(size_t g) const {
    size_t lo = 0, hi = n;   // change of op g: last c with opBase[c] <= g (changes without ops share a base with the next)
    while (hi - lo > 1) { const size_t mid = (lo + hi) / 2; if (opBase[mid] <= g) lo = mid; else hi = mid; }
    size_t c = lo; while (c + 1 < n && opBase[c + 1] <= g) c++;
    const u32 na = nActors[c]; const ActorRef* tab = actors + actorBase[c];
    const u32 shift = (u32)(bytesOff + byteBase[c]) - chOff[c];
    OpRec o;
    o.objActor = rows.objActor[g]; o.objCtr = rows.objCtr[g]; o.keyActor = rows.keyActor[g]; o.keyCtr = rows.keyCtr[g];
    o.keyStrLen = rows.keyStrLen[g]; o.keyStrOff = o.keyStrLen == NULL32 ? 0 : rows.keyStrOff[g] + shift;
    o.insert = rows.insert[g]; o.action = rows.action[g]; o.valLen = rows.valLen[g]; o.valOff = rows.valOff[g] + shift;
    o.chldActor = chldActor[g]; o.chldCtr = chldCtr[g]; o.predFirst = rows.predOff[g]; o.predNum = rows.predNum[g]; o.change = (u32)c; o.pad = 0;
    ops[g] = o;
    for (u32 j = 0; j < o.predNum; j++) { preds[2 * (size_t)(o.predFirst + j)] = rows.predActor[o.predFirst + j]; preds[2 * (size_t)(o.predFirst + j) + 1] = rows.predCtr[o.predFirst + j]; }
    // in the reference's order: object, key, value, child, preds
    if (o.objCtr != NULL32 && o.objActor != NULL32 && o.objActor >= na) { raise(err, DE_OBJ_ACTOR, g); return; }
    const bool keyStr = o.keyStrLen != NULL32 && o.keyStrLen != 0;
    if (!keyStr && o.keyCtr != 0 && o.keyActor != NULL32 && o.keyActor >= na) { raise(err, DE_KEY_ACTOR, g); return; }
    const u32 vl = o.valLen == NULL32 ? 0u : o.valLen, vr = CX_VAL_RAW;
    const u64 rawEnd = (u64)colOff[(size_t)vr * n + c] + colLen[(size_t)vr * n + c];
    if ((u64)rows.valOff[g] + (vl >> 4) > rawEnd) { raise(err, KE_SUBARRAY, g); return; }
    if (vl > 2) { if (const u32 e = decode_value_error(arena, vl, rows.valOff[g])) { raise(err, e, g); return; } }
    if (o.chldActor != NULL32 && o.chldActor >= na) { raise(err, DE_CHLD_ACTOR, g); return; }
    const bool ctrSet = o.chldCtr != NULL32 && o.chldCtr != 0, actorSet = o.chldActor != NULL32 && tab[o.chldActor].len > 0;
    if (ctrSet != actorSet) { raise(err, DE_CHLD_MISMATCH, g); return; }
    for (u32 j = 0; j < o.predNum; j++) { const u32 a = rows.predActor[o.predFirst + j]; if (a != NULL32 && a >= na) { raise(err, DE_PRED_ACTOR, g); return; } }
    for (u32 j = 1; j < o.predNum; j++) {
      const u32 pa = rows.predActor[o.predFirst + j - 1], pc = rows.predCtr[o.predFirst + j - 1], ca = rows.predActor[o.predFirst + j], cc = rows.predCtr[o.predFirst + j];
      if (pc == NULL32 || cc == NULL32) { raise(err, DE_PRED_NULL, g); return; }
      if (pc < cc) continue;
      if (pc > cc) { raise(err, DE_PRED_ORDER, g); return; }
      if (pa == NULL32 || ca == NULL32) { raise(err, DE_PRED_NULL, g); return; }
      if (chg_actor_cmp(table, tab[pa], tab[ca]) >= 0) { raise(err, DE_PRED_ORDER, g); return; }
    }
  }
};

}  // namespace amg
