// amgpu — Engine::applyChanges / getPatch pipeline (see engine.cuh for the state layout).
#pragma once
#include "engine.cuh"
#include "misc.cuh"

namespace amg {

#ifdef AMG_EMU
#define CUDA_CHECK_EMU(x) do {} while (0)
#else
#define CUDA_CHECK_EMU(x) CUDA_CHECK(x)
#endif
static const size_t PATCH_HDR_WORDS = 20;

inline void parallel_copy(u8* dst, const u8* src, size_t n) {
  if (n < (4u << 20)) { memcpy(dst, src, n); return; }
  unsigned nt = std::min<unsigned>(8, std::max(1u, std::thread::hardware_concurrency()));
  std::vector<std::thread> ts; size_t per = (n + nt - 1) / nt;
  for (unsigned t = 0; t < nt; t++) { size_t a = t * per, b = std::min(n, a + per); if (a < b) ts.emplace_back([=] { memcpy(dst + a, src + a, b - a); }); }
  for (auto& t : ts) t.join();
}

// changes [c0, c1) of a pointer array, back to back into dst (the shape Backend.applyChanges(state, Uint8Array[]) hands over)
// (a thread's loop asks for the buffers a few changes ahead - the sources are scattered heap objects, every one a cache miss)
inline void gather_range(u8* q, const u8* const* bufs, const size_t* lens, size_t a, size_t b) {
  for (size_t i = a; i < b; i++) {
    if (i + 8 < b) { __builtin_prefetch(bufs[i + 8]); __builtin_prefetch(bufs[i + 8] + 64); }
    memcpy(q, bufs[i], lens[i]); q += lens[i];
  }
}
inline void parallel_gather(u8* dst, const u8* const* bufs, const size_t* lens, size_t c0, size_t c1) {
  size_t bytes = 0; for (size_t i = c0; i < c1; i++) bytes += lens[i];
  unsigned nt = bytes < (4u << 20) ? 1u : std::min<unsigned>(16, std::max(1u, std::thread::hardware_concurrency() / 2));   // small scattered buffers: bound by cache misses, not by bandwidth
  if (nt == 1) { gather_range(dst, bufs, lens, c0, c1); return; }
  std::vector<std::thread> ts; const size_t per = (c1 - c0 + nt - 1) / nt; size_t at = 0;
  for (unsigned t = 0; t < nt; t++) {
    const size_t a = c0 + t * per, b = std::min(c1, a + per); if (a >= b) break;
    u8* d = dst + at; for (size_t i = a; i < b; i++) at += lens[i];
    ts.emplace_back([=] { gather_range(d, bufs, lens, a, b); });
  }
  for (auto& t : ts) t.join();
}

inline void Engine::fillPatchHeader(PatchOut& out) {
  out.maxOp = st.maxOp; out.pendingChanges = queue.size();
  out.clock.clear(); for (size_t a = 0; a < st.clock.size(); a++) if (st.clock[a] > 0) out.clock.emplace_back((u32)a, st.clock[a]);
  out.deps = st.heads; out.actors = st.actorIds;
}

// writes the header and the small sections (actor, actors, clock, deps) after the big record sections
inline void Engine::finishPatch(PatchOut& out) {
  if (out.bigEnd == 0) { out.propsOff = out.editsOff = PATCH_HDR_WORDS * 8; out.elemOff = 0; out.valBytesOff = out.valBytesLen = 0; out.bigEnd = PATCH_HDR_WORDS * 8; }
  size_t small = 64 + out.actor.size(); for (auto& a : out.actors) small += 8 + a.size(); small += out.clock.size() * 16 + out.deps.size() * 32 + 64;
  patchBuf.ensure(out.bigEnd + small);   // growth preserves what is already there
  u8* b = patchBuf.p; size_t at = out.bigEnd;
  for (size_t i = out.valBytesOff + out.valBytesLen; i < out.bigEnd; i++) b[i] = 0;   // the bytes section's padding: equal patches are equal bytes
  auto pad8 = [&]() { while (at % 8) b[at++] = 0; };
  u64 hdr[PATCH_HDR_WORDS] = {0}; hdr[0] = 0x31504747414d41ULL; hdr[1] = out.maxOp; hdr[2] = out.pendingChanges; hdr[3] = out.hasActorSeq ? 1 : 0; hdr[4] = out.seq;
  pad8(); hdr[5] = at; hdr[6] = out.actor.size(); memcpy(b + at, out.actor.data(), out.actor.size()); at += out.actor.size(); pad8();
  hdr[7] = at; hdr[8] = out.actors.size();
  for (auto& a : out.actors) { const u32 l = (u32)a.size(); memcpy(b + at, &l, 4); at += 4; memcpy(b + at, a.data(), l); at += l; while (at % 4) b[at++] = 0; }
  pad8(); hdr[9] = at; hdr[10] = out.clock.size();
  for (auto& c : out.clock) { const u64 a = c.first, s = c.second; memcpy(b + at, &a, 8); memcpy(b + at + 8, &s, 8); at += 16; }
  hdr[11] = at; hdr[12] = out.deps.size(); for (auto& d : out.deps) { memcpy(b + at, d.data(), 32); at += 32; }
  hdr[13] = out.propsOff; hdr[14] = out.numProps; hdr[15] = out.editsOff; hdr[16] = out.numEdits; hdr[17] = out.elemOff; hdr[18] = out.valBytesOff; hdr[19] = out.valBytesLen;
  memcpy(b, hdr, sizeof(hdr));
  out.bytes = b; out.bytesLen = at;
}

// forgets the document but keeps every allocation (steady-state serving / benchmarking)
inline void Engine::reset() {
  sync(ctx); loaded = LoadedDoc(); unknownCols.clear();
  arenaLen = 0; hostArena.len = 0; numApplied = 0; numRows = 0; numSucc = 0; dev_memset(ctx, succOff.p, 0, 4);
  st = DocState(); changes.clear(); deflatedOriginal.clear(); deflateOnExport.clear();
  queue.clear(); queueOriginal.clear(); graph = ChangeGraph(); graphInputs.clear(); rebuildActorTable();
}

// After Backend.load the hashes of the loaded changes are unknown until computeHashGraph has run. Like the reference
// (new.js:1833-1840) the first attempt goes without them; if a change then stays unapplied (or looks out of sequence)
// because it refers to history, the hash graph is computed and the call starts over. Nothing was committed by then.
struct NeedHistory {};
inline void Engine::applyChanges(const u8* const* bufs, const size_t* lens, size_t n, const u8* blob, const u64* offsets, bool isLocal, bool wantPatch, PatchOut& out,
                                 const u8* exportMarks) {
  auto once = [&]() { ApplyCall a{bufs, lens, n, blob, offsets, isLocal, wantPatch, exportMarks}; applyChangesOnce(a, out); };
  try { once(); return; }
  catch (NeedHistory&) {}
  catch (Error& e) { if (loaded.haveHashGraph || e.code != AMG_ERR_RANGE) throw; }
  drop_peeks(ctx);
  computeHashGraph();
  out = PatchOut();
  once();
}

// One attempt at a batch: the pipeline phases of DESIGN.md section 3, in order. The kernels write scratch only; nothing
// persistent changes before commit(), and the guards restore the host side when a phase throws.
inline void Engine::applyChangesOnce(ApplyCall& a, PatchOut& out) {
  trace.begin("upload+hash+decode");
  struct EndTrace { Trace& t; ~EndTrace() { t.end(); } } endTrace{trace};
  a.arenaLen0 = a.cur = arenaLen; a.Bq = queue.size(); a.B = a.n + a.Bq;
  for (const HostChange& q : queue) a.queueBytes += q.len;
  if (a.blob && a.n > 0) a.total = a.offsets[a.n] - a.offsets[0]; else for (size_t i = 0; i < a.n; i++) a.total += a.lens[i];
  if ((u64)a.arenaLen0 + a.total + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per document");
  struct Rollback { Engine* e; size_t len; bool armed = true; ~Rollback() { if (armed) { if (e->hostArena.size() > len) e->hostArena.resize(len); e->rebuildActorTable(); } } } rb{this, hostArena.size()};
  struct CopyJoin { Ctx& c; ~CopyJoin() { copy_join(c); } } copyJoin{ctx};   // nothing of this call is left on the copy stream, also on the error paths
  struct SideJoin { Ctx& c; ~SideJoin() { side_join(c); } } sideJoin{ctx};   // whatever this call put on the side stream is ordered before the next call
  if (a.B == 0) { rb.armed = false; fillPatchHeader(out); finishPatch(out); return; }
  stageBatch(a);   trace.phase("inflate+decode-finish");
  inflateBatch(a); trace.phase("gate");
  runGate(a);      trace.phase("actors+seq+finalize");
  if (a.numNew > 0) {
    internActors(a); checkSequence(a); finalizeOps(a); trace.phase("opset");
    orderOpSet(a);                                      trace.phase("patch");
    if (a.wantPatch) {   // incremental patch
      objPos.ensure(ctx, a.N + 1);
      foreach(ctx, a.N, ObjPosKernel{perm.p, objRow.p, pos.p, objPos.p});
      buildPatch(PatchInputs{sorted.view(), a.N, false, newSuccOff.p, newSucc.p, succCnt.p, a.ord, &a.ops, a.M, &a.idt, rowOfOp.p, pos.p,
                             newSuccCnt.p, firstNewSucc.p, newSuccTime.p, objPos.p, pass.p, a.w}, out);
    }
    checkErr();                                         trace.phase("heads+commit");
    computeHeads(a);
  }
  commit(a); rb.armed = false;
  side_join(ctx); sync(ctx); trace.phase(nullptr);
  fillPatchHeader(out);
  if (a.isLocal && a.n == 1) {   // new.js:1874-1877
    std::vector<ChangeHot> m0(1); d2h(ctx, m0.data(), hot.p, sizeof(ChangeHot)); sync(ctx);
    out.hasActorSeq = true; out.actor.assign(m0[0].actorLen, '\0'); out.seq = m0[0].seq;
    if (m0[0].actorLen) { d2h(ctx, &out.actor[0], arena.p + m0[0].actorOff, m0[0].actorLen); sync(ctx); }
  }
  trace.mark("commit:end");
  lastB = a.B; lastM = a.M; lastP = a.P; lastBytes = a.cur - a.arenaLen0;
  finishPatch(out); trace.mark("call:patch-finished");
  trace.collect(); trace.mark("call:timers-collected");
}

// ------------------------------------------------------------ 1. stage the batch in the arena; hash and decode it piece by piece
// The change bytes go to the device in pieces on the copy stream; as soon as a piece has landed, its changes are hashed
// (side stream) and decoded (main stream) while the next piece is still crossing PCIe - both kernels read the piece
// while it is hot in L2. The host keeps NO copy of bytes that came from a pinned or device buffer of the caller: the
// mirror (hostArena) is filled lazily when something asks for it (getChanges, amg_arena ...; ensureHostMirror). Bytes
// that have to be staged through pinned memory anyway (pageable caller buffers, pointer arrays) are staged through the
// mirror itself, which then stays complete for free.
inline void Engine::stageBatch(ApplyCall& a) {
  const size_t n = a.n, B = a.B, Bq = a.Bq, arenaLen0 = a.arenaLen0, total = a.total; const u64* offsets = a.offsets;
#ifndef AMG_EMU
  if (a.blob && n > 0) { cudaPointerAttributes at; if (cudaPointerGetAttributes(&at, a.blob) == cudaSuccess) { if (at.type == cudaMemoryTypeHost) a.srcKind = a.SRC_PINNED; else if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) a.srcKind = a.SRC_DEVICE; } else cudaGetLastError(); }
#endif
  if (a.srcKind == a.SRC_PAGEABLE && total > 0) { ensureHostMirror(); hostArena.resize(arenaLen0 + total); }
  arena.ensure(ctx, arenaLen0 + total + 64, arenaLen0);
  trace.mark("stage:begin");
  batchStore.clear();   // member: the 8 MB of a 1M-change batch keep their pages across calls
  // Pieces end on change boundaries. The copies of a pinned / device buffer are queued first (they need nothing but byte
  // ranges); the (offset, length) table of the changes is built and uploaded while they run; then every piece's kernels
  // are queued behind its copy. Pageable input is staged piece by piece, each piece's kernels right behind it.
  const size_t kPiece = 16u << 20;
  pairStage.ensure(B + 1); HostChange* pairs = a.pairs = pairStage.p;   // pinned: the table goes up by DMA while the host carries on
  if (a.blob && n > 0) {
    const size_t base = offsets[0];
    // cut points: every kPiece bytes, the tail halved three more times - what is left to hash and decode once the last byte
    // has arrived is a piece of a few MB, not a whole one
    std::vector<size_t> cuts; size_t o = kPiece;
    for (; o < total && total - o > kPiece; o += kPiece) cuts.push_back(o);
    if (total > 0) { const size_t from = o - kPiece; size_t rest = total - from; for (int k = 0; k < 3 && rest > (2u << 20); k++) { rest /= 2; cuts.push_back(total - rest); } }
    size_t lastCe = 0;
    for (size_t c : cuts) {
      const size_t ce = (size_t)(std::upper_bound(offsets, offsets + n + 1, (u64)(base + c)) - offsets) - 1;   // changes that end inside the first c bytes
      if (ce <= lastCe || ce >= n) continue;
      a.pieces.push_back({(size_t)(offsets[ce] - base), ce, 0}); lastCe = ce;
    }
    a.pieces.push_back({total, n, 0});
  } else {
    size_t at = 0, nextCut = kPiece;
    for (size_t i = 0; i < n; i++) {
      pairs[i] = HostChange{(u32)(arenaLen0 + at), (u32)a.lens[i]}; at += a.lens[i];
      if (at >= nextCut && i + 1 < n) { a.pieces.push_back({at, i + 1, 0}); nextCut = at + kPiece; }
    }
    a.pieces.push_back({at, n, 0});
  }
  a.cur = arenaLen0 + total;
  copy_fork(ctx);   // the copy stream starts behind what is queued on the main stream so far (arena growth)
  a.copiesFirst = a.srcKind != a.SRC_PAGEABLE;
  if (a.copiesFirst) { size_t byte0 = 0, ch0 = 0; for (auto& pc : a.pieces) { queueCopy(a, pc, byte0, ch0); byte0 = pc.byteEnd; ch0 = pc.changeEnd; } }
  trace.mark("stage:copies-queued");
  // The (offset, length) table of the changes. Packed batch whose offsets array is pinned or device memory: the array goes
  // up by DMA and a kernel derives the table (the host's own copy is filled later, in the shadow of the device work).
  // Otherwise the host fills a pinned table and uploads that.
#ifndef AMG_EMU
  if (a.blob && n >= 4096) { cudaPointerAttributes at; if (cudaPointerGetAttributes(&at, offsets) == cudaSuccess) a.offsetsByDma = at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged; else cudaGetLastError(); }
#endif
  for (size_t i = 0; i < Bq; i++) pairs[n + i] = queue[i];
  chPairs.ensure(ctx, B); chOff.ensure(ctx, B); chLen.ensure(ctx, B);
  if (a.offsetsByDma) {
    DBuf<u64>& offsD = offsDev; offsD.ensure(ctx, n + 2);
    CUDA_CHECK_EMU(cudaMemcpyAsync(offsD.p, offsets, (n + 1) * 8, cudaMemcpyDefault, ctx.stream));
    foreach(ctx, n, OffsetsToRangesKernel{offsD.p, (u32)(arenaLen0 - offsets[0]), chOff.p, chLen.p});
    if (Bq > 0) { h2d(ctx, chPairs.p + n, pairs + n, Bq * sizeof(HostChange)); foreach(ctx, Bq, SplitPairsKernel{chPairs.p + n, chOff.p + n, chLen.p + n}); }
  } else {
    fillPairs(a);
    h2d(ctx, chPairs.p, pairs, B * sizeof(HostChange));
    foreach(ctx, B, SplitPairsKernel{chPairs.p, chOff.p, chLen.p});
  }
  dev_memset(ctx, arena.p + a.cur, 0, 64);
  clearErr();
  hashes.ensure(ctx, (numApplied + B) * 32 + 64, numApplied * 32);
  deflList.ensure(ctx, B + 1);
  a.hashOut = hashes.p + numApplied * 32;
  a.dargs = decodeArgs(arena.p, B, a.cur - arenaLen0);
  decode_tiles_begin(ctx, a.dargs);
  trace.mark("stage:tables");
  // changes [c0, c1) are on the device once the copy stream has passed the piece's mark: hash on the side stream, decode on the main one
  auto processRange = [&](size_t c0, size_t c1, bool waitCopy, size_t mark) {
    if (c1 <= c0) return;
    if (waitCopy) copy_piece_wait(ctx, mark);   // both streams wait for the piece
    else side_fork(ctx);
    sha_range(ctx, ShaTilesArgs{arena.p, chOff.p, chLen.p, a.hashOut, errWord.p, deflList.p, (u32)c0, (u32)c1}, true);
    decode_tiles_range(ctx, a.dargs, (u32)c0, (u32)c1);
  };
  side_fork(ctx);   // the side stream is ordered behind the tables
  if (Bq > 0) processRange(n, B, false, 0);   // queue entries: their bytes are on the device already
  size_t byte0 = 0, ch0 = 0;
  for (auto& pc : a.pieces) {
    if (!a.copiesFirst) queueCopy(a, pc, byte0, ch0);
    processRange(ch0, pc.changeEnd, true, pc.mark);
    byte0 = pc.byteEnd; ch0 = pc.changeEnd;
  }
  trace.mark("stage:enqueued");
  // the host's own list of the batch entries (bookkeeping at commit, queue hand-over): a helper thread fills it while this
  // one keeps the device fed
  auto fillBatch = [this, &a]() {
    if (a.offsetsByDma) fillPairs(a);
    batchStore.assign(a.pairs, a.pairs + a.B);
    if (a.Bq > 0) { a.batchOriginal.assign(a.B, HostChange{0, 0}); for (size_t i = 0; i < a.Bq; i++) a.batchOriginal[a.n + i] = queueOriginal[i]; }
  };
  if (B >= (1u << 15)) a.fill = std::thread(fillBatch); else fillBatch();
}
inline void Engine::queueCopy(ApplyCall& a, ApplyCall::Piece& pc, size_t byte0, size_t ch0) {
  const size_t m = pc.byteEnd - byte0;
  if (m > 0) {
    u8* dst = arena.p + a.arenaLen0 + byte0; const u8* src = a.blob ? a.blob + a.offsets[0] + byte0 : nullptr;
    if (a.srcKind == a.SRC_PINNED) h2d_copy(ctx, dst, src, m);
    else if (a.srcKind == a.SRC_DEVICE) d2d_copy(ctx, dst, src, m);
    else {
      u8* stage = hostArena.data() + a.arenaLen0 + byte0;
      if (a.blob) parallel_copy(stage, src, m);
      else parallel_gather(stage, a.bufs, a.lens, ch0, pc.changeEnd);
      h2d_copy(ctx, dst, stage, m);
    }
  }
  pc.mark = copy_piece_record(ctx);
}
// the (offset, length) table of a packed batch, filled on the host (a few threads for 1M entries)
inline void Engine::fillPairs(ApplyCall& a) {
  if (!(a.blob && a.n > 0)) return;
  const size_t n = a.n; const u64* offsets = a.offsets; HostChange* pairs = a.pairs; const u32 shift = (u32)(a.arenaLen0 - offsets[0]);
  auto fill = [=](size_t lo, size_t hi) { for (size_t i = lo; i < hi; i++) { pairs[i].off = (u32)offsets[i] + shift; pairs[i].len = (u32)(offsets[i + 1] - offsets[i]); } };
  const unsigned nt = n < (1u << 16) ? 1u : std::min<unsigned>(4, std::max(1u, std::thread::hardware_concurrency()));
  if (nt == 1) fill(0, n);
  else { std::vector<std::thread> ts; const size_t per = (n + nt - 1) / nt; for (unsigned t = 0; t < nt; t++) { const size_t lo = t * per, hi = std::min(n, lo + per); if (lo < hi) ts.emplace_back(fill, lo, hi); } for (auto& t : ts) t.join(); }
}

// ------------------------------------------------------------ 2. DEFLATEd changes
// Which changes of the batch are DEFLATEd (columnar.js:742)? Those are inflated on the device, behind the batch:
// flag -> scan -> ordered list -> k_inflate (decode into scratch, sizes) -> scan -> k_inflate (assemble in place); the originals stay.
// The hash / decode kernels of the staging phase skipped them; they are hashed and decoded here, from the inflated bytes.
inline void Engine::inflateBatch(ApplyCall& a) {
  const size_t B = a.B;
  emit.ensure(ctx, B + 1); slot.ensure(ctx, B + 2);
  dev_memset(ctx, flagWord.p + 8, 0, 4);
  foreach(ctx, B, DeflateFlagKernel{arena.p, chOff.p, chLen.p, emit.p, flagWord.p + 8});
  scan_exclusive(ctx, scanTmp, emit.p, slot.p, B);
  u32 nd32 = 0, deflBytes = 0; readU32x2(slot.p + B, flagWord.p + 8, &nd32, &deflBytes);
  const size_t nd = nd32;
  trace.mark("sha:deflate-scanned");
  if (nd > 0) {
    // every stream is decoded once, into scratch (capacity: a few times its compressed size); the sizes give the places
    // behind the batch, a second kernel assembles the changes there (copy; the rare stream that did not fit is decoded again)
    foreach(ctx, B, CompactKernel{emit.p, slot.p, deflList.p});
    inflLen.ensure(ctx, nd + 1); inflOff.ensure(ctx, nd + 2); patchTriples.ensure(ctx, 2 * nd + 2); inflCap.ensure(ctx, nd + 2); inflCapOff.ensure(ctx, nd + 2); inflOvf.ensure(ctx, nd + 1);
    u32* origOff = patchTriples.p; u32* origLen = patchTriples.p + nd;
    u32 factor = 4; while (factor > 1 && (u64)factor * deflBytes + 1024ull * nd >= 0xf0000000ULL) factor--;
    const size_t scratchBytes = (size_t)factor * deflBytes + 1024 * nd + 64;
    inflScratch.ensure(ctx, scratchBytes);
    foreach(ctx, nd, InflateCapKernel{deflList.p, chLen.p, factor, inflCap.p});
    scan_exclusive(ctx, scanTmp, inflCap.p, inflCapOff.p, nd);
    InflateArgs ia{arena.p, chOff.p, chLen.p, deflList.p, nd, inflLen.p, nullptr, 0u, origOff, origLen, inflScratch.p, inflCapOff.p, inflOvf.p, errWord.p};
    const u64 extra = inflateSpeculate(ia);
    if (errSnapshot) throwKernelError(errSnapshot);   // (the error word travels with every small read)
    if ((u64)a.cur + extra + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per document");
    const size_t extraStart = a.cur; a.cur += extra;
    side_join(ctx);   // the arena may move: nothing may still be reading it
    arena.ensure(ctx, a.cur + 64, extraStart);
    ia.arena = arena.p; ia.outOff = inflOff.p; ia.extraStart = (u32)extraStart;
    inflate_changes(ctx, INFL_PLACE, ia);
    dev_memset(ctx, arena.p + a.cur, 0, 64);
    foreach(ctx, nd, InflatePatchKernel{deflList.p, inflLen.p, inflOff.p, (u32)extraStart, chOff.p, chLen.p});
    foreach(ctx, nd, ShaKernel{arena.p, chOff.p, chLen.p, a.hashOut, errWord.p, deflList.p, nullptr});
    a.inflNd = nd; a.inflExtraStart = extraStart; a.inflExtra = extra; a.inflPending = true;   // host bookkeeping happens in finishInflate()
    trace.mark("sha:inflated");
  }
  // changes the tile kernel passed on (inflated ones, changes outside their tile's window), then the totals
  { DecodeTilesArgs fin = a.dargs; fin.arena = arena.p; decode_tiles_list(ctx, fin, deflList.p, (u32)a.inflNd); decode_tiles_finish(ctx, fin, B); }
  lastDeflCount = a.inflNd; lastDeflStart = a.inflExtraStart;
  trace.mark("decode:finish-enqueued");
  side_join(ctx);
}
// The first inflate pass (sizes into ia.outLen), the places of the inflated changes behind the batch (inflOff, 32-bit scan)
// and their total. One stream may inflate to almost 2^31 bytes, so the scan wraps for two of them: the total is summed in
// 64 bits by the pass itself, and the callers refuse one past the arena limit before anything is placed.
inline u64 Engine::inflateSpeculate(InflateArgs& ia) {
  inflTotal.ensure(ctx, 1); dev_memset(ctx, inflTotal.p, 0, 8); ia.total = inflTotal.p;
  inflate_changes(ctx, INFL_SPECULATE, ia);
  scan_exclusive(ctx, scanTmp, ia.outLen, inflOff.p, ia.nd);
  u64 total = 0; void* dst[1] = {&total}; readWords({{inflTotal.p, 8}}, dst);
  return total;
}
// Host side of the device inflate: which batch entries moved where. Not on the critical path: runs when the information
// is first needed (queue hand-over, commit).
inline void Engine::ApplyCall::finishInflate(Engine& e) {
  if (!inflPending) return;
  inflPending = false; const size_t nd = inflNd; Ctx& ctx = e.ctx;
  u32* origOff = e.patchTriples.p; u32* origLen = e.patchTriples.p + nd;
  e.pinnedScratch.ensure(5 * nd + 16); u32* ps = e.pinnedScratch.p;   // pinned: the five small copies queue up and complete with one sync
  d2h(ctx, ps, e.deflList.p, nd * 4); d2h(ctx, ps + nd, e.inflLen.p, nd * 4); d2h(ctx, ps + 2 * nd, e.inflOff.p, nd * 4);
  d2h(ctx, ps + 3 * nd, origOff, nd * 4); d2h(ctx, ps + 4 * nd, origLen, nd * 4);
  if (e.hostArena.size() == inflExtraStart) {   // the mirror is complete up to here: keep it complete
    e.hostArena.resize(inflExtraStart + inflExtra);
    d2h(ctx, e.hostArena.data() + inflExtraStart, e.arena.p + inflExtraStart, inflExtra);
  }
  sync(ctx);
  deflIdx.assign(ps, ps + nd); inflOrig.resize(nd);   // deflIdx is ascending: (batch index, original range), looked up by binary search
  for (size_t k = 0; k < nd; k++) { const u32 bi = ps[k]; inflOrig[k] = HostChange{ps[3 * nd + k], ps[4 * nd + k]}; e.batchStore[bi] = HostChange{(u32)inflExtraStart + ps[2 * nd + k], ps[nd + k]}; }
}
inline HostChange Engine::ApplyCall::originalOf(size_t b) const {
  if (!batchOriginal.empty() && batchOriginal[b].len) return batchOriginal[b];
  auto it = std::lower_bound(deflIdx.begin(), deflIdx.end(), (u32)b);
  return it != deflIdx.end() && *it == (u32)b ? inflOrig[it - deflIdx.begin()] : HostChange{0, 0};
}

// hashTable holding g for hash g of hashes [0, count) (for repeated hashes the smallest g)
inline u64 Engine::hashTableOf(const u8* hs, size_t count) {
  const size_t tcap = pow2_at_least(2 * count + 2);
  hashTable.ensure(ctx, tcap); dev_memset(ctx, hashTable.p, 0xff, tcap * 4);
  foreach(ctx, count, HashInsertKernel{hs, hashTable.p, (u64)tcap - 1});
  return (u64)tcap - 1;
}

// ------------------------------------------------------------ 3. causal gate
// (parse errors surface with the first host round trip of the gate: the error word travels with every small read, and a
//  change that failed to parse has zero deps / ops so the kernels in between have nothing to walk)
inline void Engine::runGate(ApplyCall& a) {
  const size_t B = a.B;
  depBase.ensure(ctx, B + 1); scan_exclusive(ctx, scanTmp, nDeps.p, depBase.p, B);
  // every dependency occupies 32 bytes of its change, and every entry's bytes are this call's or a queued entry's: a bound
  // instead of a read of the exact total
  const size_t depBound = (a.cur - a.arenaLen0 + a.queueBytes) / 32 + B + 1;
  depIdx.ensure(ctx, depBound + 1); primary.ensure(ctx, B); pass.ensure(ctx, B);
  a.G = numApplied + B; const u64 mask = hashTableOf(hashes.p, a.G);
  foreach(ctx, B, ResolveDepsKernel{arena.p, hashes.p, hashTable.p, mask, hot.p, nDeps.p, numApplied, depBase.p, depIdx.p, primary.p});
  fill32(pass.p, 1, B);
  dev_memset(ctx, flagWord.p + 12, 0, 4);
  foreach(ctx, B, GateDupFlagKernel{primary.p, numApplied, flagWord.p + 12});
  bool copiesChecked = false, haveCopies = false; u32* decTot = a.decTot;
  for (size_t iter = 0; iter <= B + 1; iter += 2) {   // two sweeps per host round trip: the common batch settles in the first
    if (haveCopies) break;
    foreach(ctx, B, RelaxKernel{depBase.p, depIdx.p, nDeps.p, primary.p, numApplied, pass.p, flagWord.p, (u32)B + 1});
    dev_memset(ctx, flagWord.p, 0, 4);
    foreach(ctx, B, RelaxKernel{depBase.p, depIdx.p, nDeps.p, primary.p, numApplied, pass.p, flagWord.p, (u32)B + 1});
    u32 again = 0, copies = 0;
    { void* dst[7] = {&again, &copies, &decTot[0], &decTot[1], &decTot[2], &decTot[3], &a.D};   // a.D: the batch's dependency count (change graph)
      readWords({{flagWord.p, 4}, {flagWord.p + 12, 4}, {decTotalsPtr(), 4}, {decTotalsPtr() + 1, 4}, {decTotalsPtr() + 2, 4}, {decTotalsPtr() + 3, 4}, {depBase.p + B, 4}}, dst); }
    checkErr();   // free: the error word came with the read
    if (iter == 0 && decodeOverflowed(decTot)) {   // the raw row tables were too small for this batch: grown, decoded again (same results otherwise)
      runDecodeTiles(arena.p, B, a.cur - a.arenaLen0, deflList.p, a.inflNd, a.inflExtraStart);   // the whole batch is resident by now (inflated changes re-pointed)
      void* d2[4] = {&decTot[0], &decTot[1], &decTot[2], &decTot[3]};
      readWords({{decTotalsPtr(), 4}, {decTotalsPtr() + 1, 4}, {decTotalsPtr() + 2, 4}, {decTotalsPtr() + 3, 4}}, d2);
      if (decTot[2]) throw Error(AMG_ERR_INTERNAL, "amgpu: decode row tables overflowed twice");
    }
    if (!copiesChecked) { copiesChecked = true; haveCopies = copies != 0; }
    if (!again) break;
  }
  if (haveCopies) {   // rare: a change that is waiting was delivered again (gate.cuh, GateBestKernel ...)
    gateBest.ensure(ctx, B + 1); fill32(pass.p, 1, B);
    for (size_t iter = 0; iter <= B + 1; iter++) {
      dev_memset(ctx, gateBest.p, 0xff, B * 8); dev_memset(ctx, flagWord.p, 0, 4);
      foreach(ctx, B, GateBestKernel{primary.p, pass.p, numApplied, gateBest.p});
      foreach(ctx, B, RelaxCopiesKernel{depBase.p, depIdx.p, nDeps.p, primary.p, numApplied, gateBest.p, pass.p, flagWord.p, (u32)B + 1});
      const u32 again = readU32(flagWord.p);
      checkErr();
      if (!again) break;
    }
    dev_memset(ctx, gateBest.p, 0xff, B * 8);
    foreach(ctx, B, GateBestKernel{primary.p, pass.p, numApplied, gateBest.p});
    const size_t depTotal = readU32(depBase.p + B);
    if (depTotal) foreach(ctx, depTotal, GateDepWinnerKernel{gateBest.p, numApplied, depIdx.p});
    foreach(ctx, B, GateWinnerKernel{gateBest.p, numApplied, primary.p});
  }
  trace.mark("gate:settled");
  applied.ensure(ctx, B); appRank.ensure(ctx, B + 1); isRow.ensure(ctx, B + 1);
  dev_memset(ctx, flagWord.p, 0, 8);
  foreach(ctx, B, AppliedFlagKernel{primary.p, pass.p, numApplied, applied.p, isRow.p, flagWord.p});
  u32 stats[2]; readU32x2(flagWord.p, flagWord.p + 1, &stats[0], &stats[1]);
  a.numNew = stats[0]; a.inOrder = stats[1] <= 1;
  if (a.inOrder) scan_exclusive(ctx, scanTmp, isRow.p, appRank.p, B);
  else {
    sortKeys.ensure(ctx, B); sortVals.ensure(ctx, B);
    foreach(ctx, B, PassKeyKernel{pass.p, applied.p, sortKeys.p, sortVals.p});
    sortPairs(sortKeys, sortVals, B, 32);
    foreach(ctx, B, RankFromOrderKernel{sortVals.p, appRank.p, a.numNew});
  }
  if (a.numNew < B || !a.inOrder) {
    a.appliedH.resize(B); a.primaryH.resize(B); a.appRankH.resize(B);
    d2h(ctx, a.appliedH.data(), applied.p, B); d2h(ctx, a.primaryH.data(), primary.p, B * 4); d2h(ctx, a.appRankH.data(), appRank.p, B * 4); sync(ctx);
  }
  if (!loaded.haveHashGraph && a.numNew < B) throw NeedHistory{};   // a change waits for (or repeats) something older than the loaded heads
  // the queue after this call: every batch entry whose hash is still not applied (new.js:1569-1570, 1832)
  if (a.numNew < B) {
    a.needBatch(); a.finishInflate(*this);
    for (size_t b = 0; b < B; b++) {
      const u32 pr = a.primaryH[b];
      const bool hashApplied = pr < numApplied || a.appliedH[pr - numApplied];
      if (!hashApplied) { a.newQueue.push_back(batchStore[b]); a.newQueueOriginal.push_back(a.originalOf(b)); }
    }
  }
}

// ------------------------------------------------------------ 4. actors
inline void Engine::internActors(ApplyCall& a) {
  const size_t B = a.B; a.now = st; std::vector<std::string>& actors = a.now.actorIds;
  authorSlot.ensure(ctx, B); newSlots.ensure(ctx, B + 1); u32 fresh = 0, amapTotal = 0;
  // the actor map's place for every applied change (author + other-actor table); its exact size comes with the read below
  // (a change has fewer table entries than bytes, so the 32-bit scan cannot wrap below the 4 GiB arena limit)
  amapBase.ensure(ctx, B + 1); rowSlot.ensure(ctx, B + 1);
  foreach(ctx, B, MaskedCountKernel{nActors.p, applied.p, rowSlot.p});
  scan_exclusive(ctx, scanTmp, rowSlot.p, amapBase.p, B);
  while (true) {   // grow the table until the distinct authors fit at load factor <= 1/2
    dev_memset(ctx, flagWord.p, 0, 8);
    foreach(ctx, B, ActorInternKernel{arena.p, hot.p, applied.p, appRank.p, actorSlots.p, (u64)actorCap - 1, authorSlot.p, flagWord.p + 1});
    foreach(ctx, B, NewActorKernel{hot.p, applied.p, authorSlot.p, actorSlots.p, newSlots.p, flagWord.p});
    u32 full = 0; { void* dst[3] = {&fresh, &full, &amapTotal}; readWords({{flagWord.p, 4}, {flagWord.p + 1, 4}, {amapBase.p + B, 4}}, dst); }
    if (!full && (actors.size() + fresh) * 2 <= actorCap) break;
    actorCap *= 4; actorSlots.ensure(ctx, actorCap); rebuildActorTable();
  }
  if (fresh > 0) {
    trace.mark("actors:interned");
    // slot numbers, slot records and id bytes of the new actors in ONE round trip (gathered into a staging buffer)
    static const u32 ACTOR_STAGE = 64;
    hashTmp.ensure(ctx, (size_t)fresh * (4 + sizeof(ActorSlot) + ACTOR_STAGE) + 64);
    u8* stageD = hashTmp.p; const size_t recsAt = ((size_t)fresh * 4 + 15) & ~(size_t)15, bytesAt = recsAt + (size_t)fresh * sizeof(ActorSlot), stageLen = bytesAt + (size_t)fresh * ACTOR_STAGE;
    foreach(ctx, fresh, GatherNewActorsKernel{arena.p, actorSlots.p, newSlots.p, reinterpret_cast<u32*>(stageD), reinterpret_cast<ActorSlot*>(stageD + recsAt), stageD + bytesAt, ACTOR_STAGE});
    std::vector<u8> stageH(stageLen); d2h(ctx, stageH.data(), stageD, stageLen); sync(ctx);
    std::vector<u32> slotsH(fresh); memcpy(slotsH.data(), stageH.data(), (size_t)fresh * 4);
    std::vector<ActorSlot> recs(fresh); memcpy(recs.data(), stageH.data() + recsAt, (size_t)fresh * sizeof(ActorSlot));
    std::vector<u32> order(fresh); for (u32 i = 0; i < fresh; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](u32 x, u32 y) { return recs[x].first < recs[y].first; });
    std::vector<u32> ids(fresh), nums(fresh); actors.reserve(actors.size() + fresh);   // async copies target the strings: no reallocation below
    bool longIds = false;
    for (u32 k = 0; k < fresh; k++) {
      const ActorSlot& r = recs[order[k]]; ids[k] = slotsH[order[k]]; nums[k] = (u32)actors.size();
      actors.emplace_back(r.repLen, '\0');
      if (r.repLen <= ACTOR_STAGE) memcpy(&actors.back()[0], stageH.data() + bytesAt + (size_t)order[k] * ACTOR_STAGE, r.repLen);
      else { d2h(ctx, &actors.back()[0], arena.p + r.repOff, r.repLen); longIds = true; }   // from the device copy: the host mirror may still be filling
      a.now.actorRep.emplace_back(r.repOff, r.repLen);
    }
    if (longIds) sync(ctx);
    if (actors.size() > 65535) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 65535 actors in one document");
    sortVals.ensure(ctx, 2 * fresh); h2d(ctx, sortVals.p, ids.data(), fresh * 4); h2d(ctx, sortVals.p + fresh, nums.data(), fresh * 4);
    foreach(ctx, fresh, SetActorNumKernel{actorSlots.p, sortVals.p, sortVals.p + fresh});
  }
  const size_t A = actors.size(); a.now.clock.resize(A, 0);
  {   // rank of every actor in hex-string order (== byte order of the raw ids; new.js:64-65, 1180, 1198)
    std::vector<u32> order(A), rank(A); for (size_t i = 0; i < A; i++) order[i] = (u32)i;
    std::sort(order.begin(), order.end(), [&](u32 x, u32 y) { return actors[x] < actors[y]; });
    for (size_t i = 0; i < A; i++) rank[order[i]] = (u32)i;
    actorRank.ensure(ctx, A + 1); h2d(ctx, actorRank.p, rank.data(), A * 4);
  }
  a.ord = Ord{actorRank.p, bits_for(A > 1 ? A - 1 : 1)};
  trace.mark("actors:numbered");
  amap.ensure(ctx, (size_t)amapTotal + 1);   // exact: an other-actor table entry can be a single byte (an empty id)
  foreach(ctx, B, ActorMapKernel{arena.p, hot.p, nActors.p, applied.p, appRank.p, actorSlots.p, (u64)actorCap - 1, amapBase.p, amap.p, errWord.p});
  trace.mark("actors:mapped");
}

// ------------------------------------------------------------ 5. sequence numbers
inline void Engine::checkSequence(ApplyCall& a) {
  const size_t B = a.B, A = a.now.actorIds.size();
  changeActor.ensure(ctx, B); actorCnt.ensure(ctx, A + 1); actorBaseD.ensure(ctx, A + 1); seqSlot.ensure(ctx, a.numNew + 1);
  dev_memset(ctx, actorCnt.p, 0, (A + 1) * 4);
  foreach(ctx, B, ChangeActorKernel{amapBase.p, amap.p, applied.p, changeActor.p, actorCnt.p});
  if (const u64 ew = fetchErr()) throwActorError(ew, a.now.actorIds);
  scan_exclusive(ctx, scanTmp, actorCnt.p, actorBaseD.p, A);
  DBuf<u64>& clockDev = pairKey;   // scratch reuse before the succ phase
  clockDev.ensure(ctx, A + 1); h2d(ctx, clockDev.p, a.now.clock.data(), A * 8);
  dev_memset(ctx, seqSlot.p, 0xff, (a.numNew + 1) * 4); dev_memset(ctx, flagWord.p, 0, 4);
  lastChangeNext.ensure(ctx, A + 1); d2d(ctx, lastChangeNext.p, lastChange.p, st.actorIds.size() * 4);   // commit() swaps it in
  foreach(ctx, B, SeqScatterKernel{hot.p, applied.p, changeActor.p, appRank.p, actorBaseD.p, actorCnt.p, clockDev.p, seqSlot.p, flagWord.p, lastChangeNext.p, (u32)numApplied});
  foreach(ctx, B, SeqMonoKernel{hot.p, applied.p, changeActor.p, actorBaseD.p, actorCnt.p, clockDev.p, seqSlot.p, flagWord.p});
  std::vector<u32> actorCntH(A); d2h(ctx, actorCntH.data(), actorCnt.p, A * 4);
  if (readU32(flagWord.p)) throwSequenceError(a);
  for (size_t x = 0; x < A; x++) a.now.clock[x] += actorCntH[x];
  trace.mark("seq:checked");
}
// an unknown actor is named like the reference does (new.js:1446): the actor table of the change the kernel reported is read again
inline void Engine::throwActorError(u64 ew, const std::vector<std::string>& actors) {
  if ((ew & 0xff) != KE_UNKNOWN_ACTOR) throwKernelError(ew);
  const size_t b = (size_t)(ew >> 8); ChangeHot m0; u32 na0 = 1; d2h(ctx, &m0, hot.p + b, sizeof(ChangeHot)); d2h(ctx, &na0, nActors.p + b, 4); sync(ctx);
  std::vector<u8> bytes(m0.len); d2h(ctx, bytes.data(), arena.p + m0.off, m0.len); sync(ctx);
  ByteReader r(bytes.data(), m0.otherOff - m0.off, m0.len); std::string culprit; bool found = false;   // (an empty id can be the culprit)
  for (u32 k = 0; k < na0 && !r.err; k++) {
    u32 off, len; if (k == 0) { off = m0.actorOff - m0.off; len = m0.actorLen; } else { len = (u32)r.uleb(); off = r.pos; r.skip(len); }
    if (r.err) break;
    const std::string id((const char*)bytes.data() + off, len);
    if (std::find(actors.begin(), actors.end(), id) == actors.end()) { culprit = id; found = true; break; }
  }
  if (found) throw Error(AMG_ERR_RANGE, "actorId " + hex_of((const u8*)culprit.data(), culprit.size()) + " is not known to document");
  throwKernelError(ew);
}
// the sequence check failed: replay it in application order on the host to produce the reference's message
inline void Engine::throwSequenceError(ApplyCall& a) {
  const size_t B = a.B; const std::vector<std::string>& actors = a.now.actorIds;
  std::vector<ChangeHot> mh(B); std::vector<u32> ca(B), ar(B); std::vector<u8> ap(B);
  d2h(ctx, mh.data(), hot.p, B * sizeof(ChangeHot)); d2h(ctx, ca.data(), changeActor.p, B * 4); d2h(ctx, ar.data(), appRank.p, B * 4); d2h(ctx, ap.data(), applied.p, B); sync(ctx);
  std::vector<u32> byRank(a.numNew, 0); for (size_t b = 0; b < B; b++) if (ap[b]) byRank[ar[b]] = (u32)b;
  std::vector<u64> clk = a.now.clock;
  for (size_t k = 0; k < a.numNew; k++) {
    const u32 b = byRank[k]; const u64 expected = clk[ca[b]] + 1; const std::string actorHex = hex_of((const u8*)actors[ca[b]].data(), actors[ca[b]].size());
    if (mh[b].seq < expected) throw Error(AMG_ERR_RANGE, "Reuse of sequence number " + std::to_string(mh[b].seq) + " for actor " + actorHex);
    if (mh[b].seq > expected) throw Error(AMG_ERR_RANGE, "Skipped sequence number " + std::to_string(expected) + " for actor " + actorHex);
    clk[ca[b]] = mh[b].seq;
  }
  throw Error(AMG_ERR_INTERNAL, "amgpu: sequence check disagreement");
}

// ------------------------------------------------------------ 6. ops of the applied changes
// The rows were decoded with the headers (staging phase), in batch order. When every change of the batch is applied the
// op / pred ranges of the changes are the raw ones; otherwise they are the scans over the applied changes only.
inline void Engine::finalizeOps(ApplyCall& a) {
  const size_t B = a.B; const u32* decTot = a.decTot;
  timeBase.ensure(ctx, B + 1);
  opBase.ensure(ctx, B + 1); predBase.ensure(ctx, B + 1);
  // first op / pred of every applied change in batch order (the raw rows themselves lie in tile arrival order, rawBase)
  if (a.numNew == B) { scan_exclusive(ctx, scanTmp, nOps.p, opBase.p, B); scan_exclusive(ctx, scanTmp, nPreds.p, predBase.p, B); a.M = decTot[0]; a.P = decTot[1]; }
  else {
    foreach(ctx, B, MaskedCountKernel{nOps.p, applied.p, rowSlot.p}); scan_exclusive(ctx, scanTmp, rowSlot.p, opBase.p, B);
    foreach(ctx, B, MaskedCountKernel{nPreds.p, applied.p, rowSlot.p}); scan_exclusive(ctx, scanTmp, rowSlot.p, predBase.p, B);
    u32 m32 = 0, p32 = 0; void* dst[2] = {&m32, &p32}; readWords({{opBase.p + B, 4}, {predBase.p + B, 4}}, dst); a.M = m32; a.P = p32;
  }
  if (decTot[0] >= 0x7fffffffu || decTot[1] >= 0x7fffffffu) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^31 operations in one call");
  trace.mark("decode:counts");
  if (!a.inOrder) {
    perm.ensure(ctx, B + 1); dev_memset(ctx, perm.p, 0, (B + 1) * 4);
    foreach(ctx, B, OpsInOrderKernel{nOps.p, applied.p, appRank.p, perm.p});
    scan_exclusive(ctx, scanTmp, perm.p, perm.p, a.numNew);
  }
  foreach(ctx, B, TimeBaseKernel{perm.p, applied.p, appRank.p, opBase.p, a.inOrder ? 1 : 0, timeBase.p});
  DBuf<u64>& maxOpD = pairSucc; maxOpD.ensure(ctx, 1); h2d(ctx, maxOpD.p, &a.now.maxOp, 8);
  foreach(ctx, B, MaxOpKernel{hot.p, nOps.p, applied.p, decErr.p, maxOpD.p, errWord.p});
  d2h(ctx, &a.now.maxOp, maxOpD.p, 8);
  RawRows raw = rawRows();
  lastNumLarge = 0;
  if (decTot[3] & 1u) {   // changes with more than SMALL_CHANGE_OPS ops: (column, change)-parallel expansion into their reserved rows
    largeFlag.ensure(ctx, B + 1); largeSlot.ensure(ctx, B + 2); largeList.ensure(ctx, B + 1);
    foreach(ctx, B, LargeFlagKernel{nOps.p, applied.p, largeFlag.p});
    scan_exclusive(ctx, scanTmp, largeFlag.p, largeSlot.p, B);
    lastNumLarge = readU32(largeSlot.p + B);
    if (lastNumLarge > 0) {
      foreach(ctx, B, CompactKernel{largeFlag.p, largeSlot.p, largeList.p});
      // bulk changes (thousands of ops in one change): their columns are expanded in parallel by the token / record
      // decoders of doccols.cuh, column by column; whatever those decline (non-canonical streams, columns that do not hold
      // exactly the op count) and all other large changes go through DecodeColumnKernel (one thread per column)
      // (hugeDone is only this batch's when decodeHugeChanges ran: otherwise it holds an earlier batch's flags)
      const bool huge = lastNumLarge <= 8;
      if (huge) decodeHugeChanges(raw, lastNumLarge);
      foreach(ctx, (size_t)NCOLS * lastNumLarge, DecodeColumnKernel{arena.p, largeList.p, lastNumLarge, hot.p, nOps.p, nPreds.p, rawBase.p, rawPredBase.p, applied.p, raw, errWord.p, huge ? hugeDone.p : nullptr});
    }
  }
  const size_t M = a.M;
  for (DBuf<u64>* b : {&o_id, &o_obj, &o_key}) b->ensure(ctx, M + 1);
  o_predId.ensure(ctx, a.P + 1);
  for (DBuf<u32>* b : {&o_keyStrOff, &o_keyStrLen, &o_flags, &o_valLen, &o_valOff, &o_predOff, &o_predNum, &o_change, &o_time}) b->ensure(ctx, M + 1);
  a.ops = OpRows{o_id.p, o_obj.p, o_key.p, o_keyStrOff.p, o_keyStrLen.p, o_flags.p, o_valLen.p, o_valOff.p, o_predOff.p, o_predNum.p, o_change.p, o_time.p, o_predId.p};
  foreach(ctx, M, FinalizeOpsKernel{B, hot.p, nActors.p, opBase.p, predBase.p, rawBase.p, rawPredBase.p, timeBase.p, amapBase.p, amap.p, applied.p, raw, a.ops, errWord.p});
  checkErr();
  trace.mark("decode:finalized");
}

// ------------------------------------------------------------ 7. op set: the new rows, RGA list order, document order, succ lists
inline void Engine::orderOpSet(ApplyCall& a) {
  const size_t M = a.M; const Ord ord = a.ord;
  if (a.now.maxOp >= (1ULL << 40)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: op counters above 2^40");
  const int ordBits = bits_for(a.now.maxOp) + ord.rb;
  isRow.ensure(ctx, M + 1); rowSlot.ensure(ctx, M + 1); rowOfOp.ensure(ctx, M + 1);
  foreach(ctx, M, RowFlagKernel{o_flags.p, isRow.p}); scan_exclusive(ctx, scanTmp, isRow.p, rowSlot.p, M);
  const size_t R = readU32(rowSlot.p + M); const size_t N = a.N = numRows + R;
  if (N >= (1u << 29)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^29 document rows");
  doc.ensure(ctx, N + 1, numRows);
  const DocRows w = a.w = doc.view();
  foreach(ctx, M, AppendRowsKernel{a.ops, isRow.p, rowSlot.p, numRows, w, rowOfOp.p});
  const size_t icap = pow2_at_least(2 * N + 2); idKeys.ensure(ctx, icap); idVals.ensure(ctx, icap); dev_memset(ctx, idKeys.p, 0, icap * 8);
  a.idt = IdTable{idKeys.p, idVals.p, (u64)icap - 1};
  foreach(ctx, N, IdInsertKernel{w.id, a.idt, errWord.p});
  objRow.ensure(ctx, N + 1); elemRow.ensure(ctx, N + 1); parentRow.ensure(ctx, N + 1);
  foreach(ctx, N, ResolveRowsKernel{w, a.idt, ord, numRows, objRow.p, elemRow.p, parentRow.p, errWord.p});
  checkErr();
  trace.mark("opset:resolved");
  // map keys: intern, verify, rank distinct keys with an LSD string sort
  const size_t kcap = pow2_at_least(2 * N + 2); keySlots.ensure(ctx, kcap); keySlot.ensure(ctx, N + 1); repList.ensure(ctx, N + 1); repCount.ensure(ctx, 4);
  foreach(ctx, kcap, KeySlotInitKernel{keySlots.p});
  foreach(ctx, N, KeyInternKernel{arena.p, w, keySlots.p, (u64)kcap - 1, keySlot.p});
  dev_memset(ctx, repCount.p, 0, 16);
  foreach(ctx, N, KeyVerifyKernel{arena.p, w, keySlots.p, keySlot.p, repList.p, repCount.p, errWord.p});
  u32 rc[2]; readU32x2(repCount.p, repCount.p + 1, &rc[0], &rc[1]);
  const size_t D = rc[0]; const u32 maxKeyLen = rc[1];
  trace.mark("opset:keys-interned");
  if (D > 0) {
    sortKeys.ensure(ctx, D); sortVals.ensure(ctx, D);
    d2d(ctx, sortVals.p, repList.p, D * 4);
    const int chunks = (int)((maxKeyLen + 6) / 7);
    for (int ch = std::max(chunks, 1) - 1; ch >= 0; ch--) {
      foreach(ctx, D, KeyChunkKernel{arena.p, w, sortVals.p, (u32)ch * 7, sortKeys.p});
      sortPairs(sortKeys, sortVals, D, 64);
    }
    foreach(ctx, D, KeyRankKernel{sortVals.p, keySlot.p, keySlots.p});
  }
  // RGA order of every list: sibling sort, Euler tour, pointer jumping
  listPos.ensure(ctx, N + 1); insItems.ensure(ctx, N + 1); emit.ensure(ctx, N + 1); slot.ensure(ctx, N + 2);
  foreach(ctx, N, InsertFlagKernel{w, emit.p}); scan_exclusive(ctx, scanTmp, emit.p, slot.p, N);
  const size_t I = readU32(slot.p + N);
  trace.mark("opset:inserts-counted");
  if (I > 0) {
    const int parentBits = bits_for(N) + 1;
    if (ordBits + parentBits > 64) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: opId range x document size exceeds the 64-bit sibling sort key");
    foreach(ctx, N, CompactKernel{emit.p, slot.p, insItems.p});
    sortKeys.ensure(ctx, I); sortVals.ensure(ctx, I);
    foreach(ctx, I, SiblingKeyKernel{w, insItems.p, parentRow.p, objRow.p, ord, ordBits, sortKeys.p, errWord.p});
    d2d(ctx, sortVals.p, insItems.p, I * 4);
    sortPairs(sortKeys, sortVals, I, ordBits + parentBits);
    checkErr();
    itemIdx.ensure(ctx, N + 1); objSlot.ensure(ctx, N + 2);
    foreach(ctx, I, ItemIndexKernel{sortVals.p, itemIdx.p});
    foreach(ctx, N, ListObjFlagKernel{w, emit.p}); scan_exclusive(ctx, scanTmp, emit.p, objSlot.p, N);
    const size_t Lo = readU32(objSlot.p + N);
    const size_t S = 2 * I + 2 * Lo; eNext.ensure(ctx, S + 1); eRank.ensure(ctx, S + 1); ePacked.ensure(ctx, S + 1); ePacked2.ensure(ctx, S + 1);
    foreach(ctx, S, EulerInitKernel{eNext.p, eRank.p});
    foreach(ctx, I, EulerLinkKernel{sortKeys.p, ordBits, itemIdx.p, objSlot.p, eNext.p, eRank.p, I});
    foreach(ctx, S, ListRankPackKernel{eNext.p, eRank.p, ePacked.p});
    const int rounds = bits_for(S);
    for (int k = 0; k < rounds; k++) {
      foreach(ctx, S, ListRankPackedKernel{ePacked.p, ePacked2.p});
      ePacked.swap(ePacked2);
    }
    foreach(ctx, S, ListRankUnpackKernel{ePacked.p, eRank.p});
    foreach(ctx, N, ListPosKernel{eRank.p, elemRow.p, objRow.p, itemIdx.p, objSlot.p, (u32)I, listPos.p});
  } else dev_memset(ctx, listPos.p, 0, (N + 1) * 4);
  checkErr();
  trace.mark("opset:list-ranked");
  // document order: stable LSD over (object, key rank | list position, opId within the key / element)
  perm.ensure(ctx, N + 1); pos.ensure(ctx, N + 1); sortKeys.ensure(ctx, N);
  foreach(ctx, N, IotaKernel{perm.p});
  const int fieldBits[3] = {ordBits + 1, bits_for(N), ordBits + 1};
  for (int f = 0; f < 3; f++) {
    foreach(ctx, N, DocKeyKernel{f, w, perm.p, listPos.p, keySlots.p, keySlot.p, ord, sortKeys.p});
    sortPairs(sortKeys, perm, N, fieldBits[f]);
  }
  foreach(ctx, N, InversePermKernel{perm.p, pos.p});
  trace.mark("opset:doc-ordered(enqueued)");
  // succ lists of the new document (old pairs re-keyed + the batch's preds), the checks on what the preds refer to, and the
  // rows gathered into document order
  const size_t numPairs = a.numPairs = numSucc + a.P;
  pairKey.ensure(ctx, numPairs + 1); pairSucc.ensure(ctx, numPairs + 1); pairIdx.ensure(ctx, numPairs + 1); pairPos.ensure(ctx, numPairs + 1); pairTime.ensure(ctx, numPairs + 1);
  foreach(ctx, M, DelElemCheckKernel{a.ops, a.idt, w, errWord.p});
  checkErr();
  foreach(ctx, numRows, OldPairsKernel{succOff.p, succ.p, pos.p, ord, pairKey.p, pairIdx.p, pairSucc.p, pairPos.p, pairTime.p});
  foreach(ctx, M, PredPairsKernel{a.ops, a.idt, pos.p, rowOfOp.p, w, elemRow.p, keySlot.p, ord, pairKey.p, pairIdx.p, pairSucc.p, pairPos.p, pairTime.p, numSucc, errWord.p});
  foreach(ctx, M, DelKeyCheckKernel{arena.p, a.ops, a.idt, w, errWord.p});
  foreach(ctx, M, IncCheckKernel{a.ops, a.idt, w, arena.p, errWord.p});
  if (const u64 ew = fetchErr()) throwOpError(ew, a.now.actorIds);
  sortPairs(pairKey, pairIdx, numPairs, ordBits);
  foreach(ctx, numPairs, PairPosKeyKernel{pairPos.p, pairIdx.p, pairKey.p});
  sortPairs(pairKey, pairIdx, numPairs, bits_for(N));
  succCnt.ensure(ctx, N + 2); newSuccCnt.ensure(ctx, N + 2); newSuccOff.ensure(ctx, N + 2); firstNewSucc.ensure(ctx, N + 2); newSucc.ensure(ctx, numPairs + 1);
  dev_memset(ctx, succCnt.p, 0, (N + 2) * 4); dev_memset(ctx, newSuccCnt.p, 0, (N + 2) * 4); dev_memset(ctx, firstNewSucc.p, 0xff, (N + 2) * 4);
  foreach(ctx, numPairs, CountSuccKernel{pairPos.p, succCnt.p});
  foreach(ctx, numPairs, NewSuccFlagKernel{pairPos.p, pairTime.p, newSuccCnt.p});
  foreach(ctx, numPairs, FirstSuccTimeKernel{pairPos.p, pairTime.p, firstNewSucc.p});
  scan_exclusive(ctx, scanTmp, succCnt.p, newSuccOff.p, N);
  newSuccTime.ensure(ctx, numPairs + 1);
  foreach(ctx, numPairs, WriteSuccKernel{pairIdx.p, pairSucc.p, newSucc.p, pairTime.p, newSuccTime.p});
  sorted.ensure(ctx, N + 1);
  foreach(ctx, N, GatherRowsKernel{w, sorted.view(), perm.p});
  trace.mark("opset:succ+gather(enqueued)");
}

// names the op of a missing pred or of an increment without a counter like the reference does
inline void Engine::throwOpError(u64 ew, const std::vector<std::string>& actors) {
  if ((ew & 0xff) == KE_PRED_MISSING) { u64 pid = 0; d2h(ctx, &pid, o_predId.p + (ew >> 8), 8); sync(ctx); throw Error(AMG_ERR_RANGE, "no matching operation for pred: " + opIdText(pid, actors)); }
  if ((ew & 0xff) == KE_UNKNOWN_COUNTER) { u64 oid = 0; d2h(ctx, &oid, o_id.p + (ew >> 8), 8); sync(ctx); throw Error(AMG_ERR_RANGE, "increment operation " + opIdText(oid, actors) + " for unknown counter"); }
  throwKernelError(ew);
}

// ------------------------------------------------------------ 9. heads
inline void Engine::computeHeads(ApplyCall& a) {
  const size_t B = a.B;
  trace.mark("commit:begin");
  DBuf<u32>& isDep = groupLinked; isDep.ensure(ctx, a.G + 1); dev_memset(ctx, isDep.p, 0, (a.G + 1) * 4);   // scratch reuse: the patch is done with it
  foreach(ctx, B, MarkDepsKernel{applied.p, nDeps.p, depBase.p, depIdx.p, isDep.p});
  emit.ensure(ctx, B + 1); slot.ensure(ctx, B + 2); objStart.ensure(ctx, B + 1);
  foreach(ctx, B, HeadFlag2Kernel{applied.p, isDep.p, numApplied, emit.p});
  scan_exclusive(ctx, scanTmp, emit.p, slot.p, B);
  foreach(ctx, B, CompactKernel{emit.p, slot.p, objStart.p});
  // one round trip for the whole answer (HeadsPackKernel); a second one only if the call leaves more heads than the block holds
  const u32 nOld = (u32)st.headIdx.size(); u32 cap = 64, nh = 0; std::vector<u32> pack;
  headsPack.ensure(ctx, nOld + 1);
  if (nOld) h2d(ctx, headsPack.p, st.headIdx.data(), nOld * 4);
  for (;;) {
    const size_t words = 1 + (size_t)nOld + 9 * (size_t)cap;
    headsOut.ensure(ctx, words + 1); pack.resize(words);
    foreach(ctx, std::max<size_t>(std::max<size_t>(nOld, cap), 1), HeadsPackKernel{slot.p + B, objStart.p, hashes.p + numApplied * 32, appRank.p, isDep.p, headsPack.p, nOld, cap, headsOut.p});
    d2h(ctx, pack.data(), headsOut.p, words * 4); sync(ctx);
    nh = pack[0];
    if (nh <= cap) break;
    cap = nh;
  }
  std::vector<std::array<u8, 32>> hs; std::vector<u32> hi;
  for (u32 i = 0; i < nOld; i++) if (!pack[1 + i]) { hs.push_back(st.heads[i]); hi.push_back(st.headIdx[i]); }
  for (u32 k = 0; k < nh; k++) { const u32* e = pack.data() + 1 + nOld + 9 * (size_t)k; std::array<u8, 32> h; memcpy(h.data(), e, 32); hs.push_back(h); hi.push_back((u32)(numApplied + e[8])); }
  std::vector<size_t> o(hs.size()); for (size_t i = 0; i < o.size(); i++) o[i] = i;
  std::sort(o.begin(), o.end(), [&](size_t x, size_t y) { return hs[x] < hs[y]; });
  a.now.heads.clear(); a.now.headIdx.clear(); for (size_t i : o) { a.now.heads.push_back(hs[i]); a.now.headIdx.push_back(hi[i]); }
}

// ------------------------------------------------------------ 10. commit (nothing before this mutated persistent state)
inline void Engine::commit(ApplyCall& a) {
  const size_t B = a.B, numNew = a.numNew;
  trace.mark("commit:heads-done");
  if (numNew > 0 && (a.decTot[3] & 2u)) collectUnknownColumns(B, a.unknownRows, a.unknownIds);   // rare: columns written by a future version (unknowncols.hpp)
  sync(ctx);
  trace.mark("commit:synced");
  a.needBatch(); a.finishInflate(*this);
  if (numNew > 0) {
    if (!(a.inOrder && numNew == B)) {   // hashes of applied changes must be contiguous in application order
      DBuf<u8>& tmp = hashTmp; tmp.ensure(ctx, numNew * 32 + 64);
      foreach(ctx, B, HashGatherKernel{hashes.p + numApplied * 32, applied.p, appRank.p, tmp.p});
      d2d(ctx, hashes.p + numApplied * 32, tmp.p, numNew * 32);
    }
    if (a.appliedH.empty()) {   // all applied, in order
      const u32 base0 = (u32)changes.size();
      if (!a.batchOriginal.empty()) for (size_t b = 0; b < B; b++) { const HostChange o = a.originalOf(b); if (o.len) deflatedOriginal.push_back({base0 + (u32)b, o}); }
      else { deflatedOriginal.reserve(deflatedOriginal.size() + a.deflIdx.size()); for (size_t k = 0; k < a.deflIdx.size(); k++) deflatedOriginal.push_back({base0 + a.deflIdx[k], a.inflOrig[k]}); }
      if (a.exportMarks) for (size_t b = 0; b < a.n; b++) if (a.exportMarks[b]) deflateOnExport.push_back(base0 + (u32)b);
      if (changes.empty()) changes.swap(batchStore); else changes.insert(changes.end(), batchStore.begin(), batchStore.end());
    } else {
      std::vector<u32> byRank(numNew);
      for (size_t b = 0; b < B; b++) if (a.appliedH[b]) byRank[a.appRankH[b]] = (u32)b;
      for (size_t k = 0; k < numNew; k++) {
        const u32 b = byRank[k];
        { const HostChange o = a.originalOf(b); if (o.len) deflatedOriginal.push_back({(u32)changes.size(), o}); }
        if (a.exportMarks && b < a.n && a.exportMarks[b]) deflateOnExport.push_back((u32)changes.size());   // only the copy that was applied carries its mark
        changes.push_back(batchStore[b]);
      }
    }
    trace.mark("commit:changes-recorded");
    doc.swap(sorted); numRows = a.N; lastChange.swap(lastChangeNext);
    succOff.swap(newSuccOff); succ.swap(newSucc); numSucc = a.numPairs;
    fill32(doc.time.p, 0, a.N);
    for (auto& kv : a.unknownRows) unknownCols.byOp[kv.first] = std::move(kv.second);
    unknownCols.colIds.insert(a.unknownIds.begin(), a.unknownIds.end());
    keepGraphInputs(a);
    loaded.bytes.clear(); numApplied += numNew; st = std::move(a.now);
    trace.mark("commit:state-swapped");
    rebuildActorTable();   // slots of actors registered in this call become permanent (first = 0)
    trace.mark("commit:actors-rebuilt");
  }
  arenaLen = a.cur; queue = a.newQueue; queueOriginal = a.newQueueOriginal;
}


// Patch emission over a document table `in.d` in document order (N rows). wholeDoc = getPatch semantics
// (new.js:1604-1635), otherwise incremental semantics for the batch `ops` (new.js:884-1040, 1461-1528).
inline void Engine::buildPatch(const PatchInputs& in, PatchOut& out) {
  const DocRows d = in.d; const size_t N = in.N, numOps = in.numOps; const bool wholeDoc = in.wholeDoc; const OpRows* ops = in.ops;
  const u32* succCntD = in.succCnt;
  out.numProps = out.numEdits = 0; out.bigEnd = 0;
  if (N == 0) return;
  // groups (map key / list element) and their visibility
  head.ensure(ctx, N + 1); headScan.ensure(ctx, N + 2); groupOf.ensure(ctx, N + 1);
  foreach(ctx, N, GroupHeadKernel{arena.p, d, head.p});
  scan_exclusive(ctx, scanTmp, head.p, headScan.p, N);
  isObjHead.ensure(ctx, N + 1); objIdx.ensure(ctx, N + 2);
  foreach(ctx, N, ObjHeadKernel{d, isObjHead.p});
  scan_exclusive(ctx, scanTmp, isObjHead.p, objIdx.p, N);
  u32 numGroups32 = 0, numObjs32 = 0; readU32x2(headScan.p + N, objIdx.p + N, &numGroups32, &numObjs32);
  const size_t numGroups = numGroups32, numObjs = numObjs32;
  groupRows.ensure(ctx, numGroups + 1); groupVisible.ensure(ctx, numGroups + 1); groupFirst.ensure(ctx, numGroups + 1); groupTouched.ensure(ctx, numGroups + 1);
  dev_memset(ctx, groupRows.p, 0, (numGroups + 1) * 4); dev_memset(ctx, groupVisible.p, 0, (numGroups + 1) * 4); dev_memset(ctx, groupTouched.p, 0, (numGroups + 1) * 4);
  groupHasChild.ensure(ctx, numGroups + 1); dev_memset(ctx, groupHasChild.p, 0, (numGroups + 1) * 4);
  foreach(ctx, N, GroupStatsKernel{headScan.p, head.p, succCntD, d, groupOf.p, groupRows.p, groupVisible.p, groupFirst.p, errWord.p, 0, groupHasChild.p});
  // objects in document order
  objStart.ensure(ctx, numObjs + 2);
  foreach(ctx, N, ObjStartKernel{isObjHead.p, objIdx.p, objStart.p, N});
  { const u32 nn = (u32)N; h2d(ctx, objStart.p + numObjs, &nn, 4); }
  emit.ensure(ctx, N + 1); marker.ensure(ctx, N + 1); slot.ensure(ctx, N + 2);
  groupLinked.ensure(ctx, std::max(numGroups, numApplied + 1) + 2);
  dev_memset(ctx, groupLinked.p, 0, (numGroups + 1) * 4);
  ListCtx lctx{d, succCntD, in.newSuccCnt, in.firstNewSucc, groupOf.p, groupFirst.p, groupRows.p, arena.p, in.succOff, in.succ, in.newSuccTime};
  MapGroupCtx mg{arena.p, ops ? *ops : OpRows{}, opAt.p, numOps, in.pass};
  bool anyListLink = false;
  auto listGroups = [&](int pass) {
    return ListGroupKernel{pass, mg, opGroupHead.p, *in.idt, in.rowOfOp, in.pos, lctx, gCount.p, gElem.p, gT1.p, gQOrd.p, nQ.p, elemHasRecs.p, elemMinT.p,
                           itemBase.p, objIdx.p, objStart.p, items.p, domTw.p, domW.p, oldVisScan.p, runHeadFlag.p, runScan.p, runStart.p, gBase.p, qIndex.p, editOut.p, editElem.p, editObjKey.p, editElemPos.p, editRowPos.p, errWord.p};
  };
  if (!wholeDoc) {
    // op groups of the batch (new.js:1085-1138), then what each list group nets out to
    nQ.ensure(ctx, N + 1); elemHasRecs.ensure(ctx, N + 1); listLinkTime.ensure(ctx, N + 1); elemMinT.ensure(ctx, N + 1);
    dev_memset(ctx, elemMinT.p, 0xff, (N + 1) * 4);
    dev_memset(ctx, nQ.p, 0, (N + 1) * 4); dev_memset(ctx, elemHasRecs.p, 0, (N + 1) * 4); dev_memset(ctx, listLinkTime.p, 0xff, (N + 1) * 4);
    if (numOps > 0) {
      opAt.ensure(ctx, numOps + 1); runHead.ensure(ctx, numOps + 1); opGroupHead.ensure(ctx, numOps + 1);
      for (DBuf<u32>* b : {&gCount, &gElem, &gT1, &gQOrd, &gBase, &qIndex}) b->ensure(ctx, numOps + 2);
      mg.opAt = opAt.p;
      foreach(ctx, numOps, OpAtTimeKernel{ops->time, opAt.p});
      foreach(ctx, numOps, RunHeadKernel{mg, runHead.p});
      foreach(ctx, numOps, GroupSplitKernel{mg, runHead.p, opGroupHead.p});
      foreach(ctx, numOps, listGroups(0));
      runHeadFlag.ensure(ctx, numOps + 1); runScan.ensure(ctx, numOps + 2); runStart.ensure(ctx, numOps + 2); elemFollower.ensure(ctx, N + 1);
      dev_memset(ctx, elemFollower.p, 0, (N + 1) * 4);
      foreach(ctx, numOps, FollowerFlagKernel{mg, opGroupHead.p, lctx, gElem.p, gT1.p, gCount.p, nQ.p, runHeadFlag.p, elemFollower.p});
      scan_exclusive(ctx, scanTmp, runHeadFlag.p, runScan.p, numOps);
      foreach(ctx, numOps, RunStartKernel{runHeadFlag.p, runScan.p, runStart.p});
      foreach(ctx, 1, RunEndKernel{runScan.p, runStart.p, (u32)numOps});
    }
    objTouchedAt.ensure(ctx, N + 1); linkDone.ensure(ctx, N + 1);
    dev_memset(ctx, objTouchedAt.p, 0xff, (N + 1) * 4); dev_memset(ctx, linkDone.p, 0xff, (N + 1) * 4); dev_memset(ctx, flagWord.p, 0, 16);
    foreach(ctx, N, TouchKernel{d, groupOf.p, in.firstNewSucc, groupTouched.p, objTouchedAt.p, in.objPos, flagWord.p + 2});
    u32 linkChanged = 1, anyLink32 = 0;
    // Three sweeps per host round trip, until a sweep changes nothing. A touch climbs at least one level of nesting per
    // sweep (a parent's make row lies below its child's rows, so a serial sweep climbs exactly one), so a fixed number of
    // rounds would leave the outer levels of deeply nested objects unlinked. It ends: objTouchedAt only decreases.
    while (linkChanged) {
      LinkKernel lk{d, groupOf.p, groupHasChild.p, groupFirst.p, groupTouched.p, in.objPos, groupLinked.p, objTouchedAt.p, flagWord.p + 2, linkDone.p, flagWord.p, listLinkTime.p, flagWord.p + 3};
      foreach(ctx, N, lk); foreach(ctx, N, lk);
      dev_memset(ctx, flagWord.p, 0, 4);
      foreach(ctx, N, lk);
      readU32x2(flagWord.p, flagWord.p + 3, &linkChanged, &anyLink32);
    }
    anyListLink = anyLink32 != 0;
  }
  // ---- map props
  DBuf<u32>& groupEmitted = elemVis;   // scratch reuse (list edits re-initialise it later)
  groupEmitted.ensure(ctx, std::max(numGroups, N) + 2); dev_memset(ctx, groupEmitted.p, 0, (numGroups + 1) * 4);
  finalTime.ensure(ctx, numGroups + 1); gBound.ensure(ctx, numGroups + 1); gFailed.ensure(ctx, numGroups + 1); memberFinal.ensure(ctx, N + 1);
  dev_memset(ctx, finalTime.p, 0, (numGroups + 1) * 4);
  if (!wholeDoc && numOps > 0) {
    dev_memset(ctx, memberFinal.p, 0, (N + 1) * 4); dev_memset(ctx, gFailed.p, 0, (numGroups + 1) * 4);
    for (int pass = 0; pass < 2; pass++)
      foreach(ctx, numOps, GroupFinalKernel{pass, mg, opGroupHead.p, *in.idt, in.rowOfOp, in.pos, groupOf.p, in.unsorted, in.ord, finalTime.p, gBound.p, gFailed.p, memberFinal.p});
  }
  counterLast.ensure(ctx, N + 1); counterTotal.ensure(ctx, N + 1); counterOwner.ensure(ctx, N + 1); dev_memset(ctx, counterOwner.p, 0xff, (N + 1) * 4);
  foreach(ctx, N, CounterKernel{arena.p, d, in.succOff, in.succ, groupOf.p, groupFirst.p, groupRows.p, counterLast.p, counterTotal.p, counterOwner.p});
  foreach(ctx, N, PropFlagKernel{d, groupOf.p, groupTouched.p, groupLinked.p, succCntD, wholeDoc ? 1 : 0, finalTime.p, gBound.p, gFailed.p, memberFinal.p, in.ord, emit.p, groupEmitted.p, counterLast.p});
  foreach(ctx, N, PropMarkerKernel{d, groupOf.p, groupTouched.p, head.p, groupEmitted.p, wholeDoc ? 1 : 0, emit.p, marker.p});
  scan_exclusive(ctx, scanTmp, emit.p, slot.p, N);
  const size_t numProps = readU32(slot.p + N);
  propOut.ensure(ctx, numProps + 1);
  foreach(ctx, N, PropEmitKernel{d, emit.p, marker.p, slot.p, propOut.p, counterLast.p, counterTotal.p});
  trace.phase("patch:list-index");
  // ---- list edits
  size_t numEdits = 0; bool shipElem = true;
  if (wholeDoc) {
    elemVis.ensure(ctx, N + 1); elemVisScan.ensure(ctx, N + 2); rowEmit.ensure(ctx, N + 1); firstVis.ensure(ctx, numGroups + 1);
    rowClass.ensure(ctx, N + 1); firstBare.ensure(ctx, numGroups + 1);
    dev_memset(ctx, firstVis.p, 0xff, (numGroups + 1) * 4); dev_memset(ctx, firstBare.p, 0xff, (numGroups + 1) * 4);
    foreach(ctx, N, ListRowClassKernel{d, groupOf.p, succCntD, counterOwner.p, rowClass.p, firstVis.p, firstBare.p});
    foreach(ctx, N, ListVisFlagKernel{d, groupOf.p, groupVisible.p, head.p, succCntD, elemVis.p, rowEmit.p, rowClass.p, firstVis.p, firstBare.p});
    scan_exclusive(ctx, scanTmp, elemVis.p, elemVisScan.p, N);
    scan_exclusive(ctx, scanTmp, rowEmit.p, slot.p, N);
    numEdits = readU32(slot.p + N);
    editOut.ensure(ctx, numEdits + 1); editElem.ensure(ctx, numEdits + 1);
    foreach(ctx, N, DocEditEmitKernel{d, rowEmit.p, slot.p, elemVisScan.p, objIdx.p, objStart.p, groupOf.p, groupFirst.p, rowClass.p, firstVis.p, firstBare.p, editOut.p, counterOwner.p, counterTotal.p});
    foreach(ctx, N, EditElemKernel{d, rowEmit.p, slot.p, groupOf.p, groupFirst.p, editElem.p});
  } else {
    size_t numGroupRecs = 0, numLink = 0, numLive = 0;
    if (numOps > 0) { scan_exclusive(ctx, scanTmp, gCount.p, gBase.p, numOps); numGroupRecs = readU32(gBase.p + numOps); }
    DBuf<u32>& elemHasLive = elemHasRecs; dev_memset(ctx, elemHasLive.p, 0, (N + 1) * 4);
    auto ensureEdits = [&](size_t n) {
      editOut.ensure(ctx, n + 1, numLive); editElem.ensure(ctx, n + 1, numLive); editObjKey.ensure(ctx, n + 1, numLive); editElemPos.ensure(ctx, n + 1);
      editOut2.ensure(ctx, n + 1); editElem2.ensure(ctx, n + 1); editElemPos2.ensure(ctx, n + 1); editObjKey2.ensure(ctx, n + 1); editRowPos.ensure(ctx, n + 1); editRowPos2.ensure(ctx, n + 1);
      sortKeys.ensure(ctx, n + 1); sortVals.ensure(ctx, n + 1);
    };
    // ---- A. records of the op groups: indexes, emission, per-object order, pops / coalescing, compaction
    if (numGroupRecs > 0) {
      // list index of a group = elements in front that were visible before the batch (one prefix sum)
      //                       + net visibility changes in front that earlier groups of the batch made (dominance count)
      nItems.ensure(ctx, N + 1); itemBase.ensure(ctx, N + 2); oldVisScan.ensure(ctx, N + 2);
      foreach(ctx, N, OldVisFlagKernel{lctx, head.p, nItems.p});
      scan_exclusive(ctx, scanTmp, nItems.p, oldVisScan.p, N);
      foreach(ctx, N, DomItemCountKernel{nQ.p, elemFollower.p, nItems.p});
      scan_exclusive(ctx, scanTmp, nItems.p, itemBase.p, N);
      const size_t T = readU32(itemBase.p + N);
      items.ensure(ctx, T + 1); items2.ensure(ctx, T + 1); zwScan.ensure(ctx, T + 2); domTw.ensure(ctx, T + 1); domTw2.ensure(ctx, T + 1); domW.ensure(ctx, T + 1); domW2.ensure(ctx, T + 1);
      foreach(ctx, numOps, listGroups(1));
      const int tbits = bits_for(numOps + 1);
#ifdef AMG_EMU
      const int localBits = 0;
#else
      const int localBits = std::min(tbits, DOM_LOCAL_BITS);   // the last levels run inside shared memory (k_dom_local)
#endif
      for (int bit = tbits - 1; bit >= localBits; bit--) {
        scan_exclusive64(ctx, scanTmp, DomScanInput{domTw.p, domW.p, bit}, zwScan.p, T);
        foreach(ctx, T, DomLevelKernel{items.p, items2.p, domTw2.p, domW2.p, zwScan.p, bit});
        items.swap(items2); domTw.swap(domTw2); domW.swap(domW2);
      }
#ifdef AMG_EMU
      foreach(ctx, T, DomResultKernel{items.p, qIndex.p});
#else
      {   // partition heads -> compact list (device-side count), then one CTA per partition
        DBuf<u32>& partFlag = domTw2; DBuf<u32>& partScan = nItems; DBuf<u32>& partHead = itemBase;   // scratch that is free by now
        partScan.ensure(ctx, T + 2); partHead.ensure(ctx, T + 2);
        foreach(ctx, T, DomPartHeadKernel{items.p, partFlag.p});
        scan_exclusive(ctx, scanTmp, partFlag.p, partScan.p, T);
        foreach(ctx, T, CompactKernel{partFlag.p, partScan.p, partHead.p});
        if (!domLocalReady) { CUDA_CHECK(cudaFuncSetAttribute(k_dom_local, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DomLocalSmem))); domLocalReady = true; }
        k_dom_local<<<ctx.numSMs * 2, 256, sizeof(DomLocalSmem), ctx.stream>>>(items.p, partHead.p, partScan.p + T, qIndex.p, localBits, errWord.p);
        CUDA_CHECK(cudaGetLastError()); ctx.launches++;
      }
#endif
      trace.phase("patch:edits+copy-out");
      ensureEdits(numGroupRecs);
      foreach(ctx, numOps, listGroups(2));
      // the records are in application order by construction: one stable sort by object gives the per-object edit lists
      foreach(ctx, numGroupRecs, EditKeyKernel{editObjKey.p, editOut.p, sortKeys.p, sortVals.p});
      sortPairs(sortKeys, sortVals, numGroupRecs, bits_for(numObjs));
      foreach(ctx, numGroupRecs, EditGatherKernel{editOut.p, editElem.p, editElemPos.p, editObjKey.p, sortVals.p, editOut2.p, editElem2.p, editElemPos2.p, editObjKey2.p});
      foreach(ctx, numGroupRecs, GatherU32Kernel{editRowPos.p, sortVals.p, editRowPos2.p});
      for (DBuf<u32>* b : {&editKind, &editPred, &editDead, &editMerge, &editMulti, &editLive}) b->ensure(ctx, numGroupRecs + 2);
      dev_memset(ctx, editDead.p, 0, (numGroupRecs + 1) * 4); dev_memset(ctx, editMulti.p, 0, (numGroupRecs + 1) * 4);
      foreach(ctx, numGroupRecs, EditFixKernel{editOut2.p, editElemPos2.p, editKind.p, editPred.p, editDead.p, numGroupRecs});
      foreach(ctx, numGroupRecs, EditMergeKernel{editOut2.p, editElem2.p, editKind.p, editPred.p, editMerge.p, editMulti.p});
      dev_memset(ctx, flagWord.p, 0, 4);
      foreach(ctx, numGroupRecs, EditLiveKernel{editDead.p, editLive.p, editOut2.p, editElem2.p, editKind.p, flagWord.p, editElemPos2.p, elemHasLive.p, editRowPos2.p, succCntD, counterLast.p});
      DBuf<u32>& liveSlot = editPred;   // pred is consumed by now
      scan_exclusive(ctx, scanTmp, editLive.p, liveSlot.p, numGroupRecs);
      u32 numLive32 = 0, needElem32 = 0; readU32x2(liveSlot.p + numGroupRecs, flagWord.p, &numLive32, &needElem32);
      numLive = numLive32; shipElem = needElem32 != 0;
      foreach(ctx, numGroupRecs, EditCompactKernel{editOut2.p, editElem2.p, editDead.p, liveSlot.p, editKind.p, editMerge.p, editMulti.p, editOut.p, editElem.p, editObjKey2.p, editObjKey.p});
    } else trace.phase("patch:edits+copy-out");
    // ---- B. setupPatches link edits on list parents: only for elements that did not keep an edit of their own; appended
    //         behind the object's other edits in the order the child objects were first touched
    if (anyListLink) {
      DBuf<u32>& linkCount = rowEmit; DBuf<u32>& linkBase = slot;
      elemVis.ensure(ctx, N + 1); elemVisScan.ensure(ctx, N + 2); linkCount.ensure(ctx, N + 1); linkBase.ensure(ctx, N + 2);
      foreach(ctx, N, ListVisFlagKernel{d, groupOf.p, groupVisible.p, head.p, succCntD, elemVis.p, linkCount.p, nullptr, nullptr, nullptr});
      scan_exclusive(ctx, scanTmp, elemVis.p, elemVisScan.p, N);   // index of a linked element = visible elements before it once the whole batch is applied
      foreach(ctx, N, ListLinkKernel{0, lctx, listLinkTime.p, elemVisScan.p, objIdx.p, objStart.p, linkCount.p, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, elemHasLive.p});
      scan_exclusive(ctx, scanTmp, linkCount.p, linkBase.p, N);
      numLink = readU32(linkBase.p + N);
      if (numLink > 0) {
        const size_t total = numLive + numLink;
        ensureEdits(total); editTime.ensure(ctx, total + 1);
        foreach(ctx, N, ListLinkKernel{1, lctx, listLinkTime.p, elemVisScan.p, objIdx.p, objStart.p, linkCount.p, linkBase.p, (u32)numLive, editOut.p, editElem.p, editObjKey.p, editElemPos.p, editTime.p, elemHasLive.p});
        // order: surviving group records as they are, then the link edits by first-touch time; then stably by object
        foreach(ctx, numLive, OffsetIotaKernel{sortVals.p, 0});
        if (numLink > 1) {
          DBuf<u64>& k2 = pairKey; DBuf<u32>& v2 = pairIdx; k2.ensure(ctx, numLink + 1); v2.ensure(ctx, numLink + 1);
          foreach(ctx, numLink, EditTimeKeyAtKernel{editTime.p, (u32)numLive, k2.p, v2.p});
          sortPairs(k2, v2, numLink, 32);
          d2d(ctx, sortVals.p + numLive, v2.p, numLink * 4);
        } else foreach(ctx, numLink, OffsetIotaKernel{sortVals.p + numLive, (u32)numLive});
        foreach(ctx, total, GatherToU64Kernel{editObjKey.p, sortVals.p, sortKeys.p});
        sortPairs(sortKeys, sortVals, total, bits_for(numObjs));
        foreach(ctx, total, EditGatherKernel{editOut.p, editElem.p, nullptr, nullptr, sortVals.p, editOut2.p, editElem2.p, nullptr, nullptr});
        editOut.swap(editOut2); editElem.swap(editElem2);
      }
    }
    numEdits = numLive + numLink;
  }
  if (wholeDoc && numEdits > 0) foreach(ctx, numEdits, RunFlagKernel{editOut.p, editElem.p, numEdits});
  out.numProps = numProps; out.numEdits = numEdits;
  out.propsOff = PATCH_HDR_WORDS * 8; out.editsOff = out.propsOff + numProps * sizeof(PropRec);
  size_t end;
  if (shipElem) { out.elemOff = out.editsOff + numEdits * sizeof(EditRec); end = out.elemOff + numEdits * 8; }
  else { out.elemOff = 0; end = out.editsOff + numEdits * sizeof(EditRec); }   // elemOff 0: every insert's elemId is its opId
  // key and value bytes of the records: gathered behind them, offsets rewritten to positions inside the patch
  const size_t nRec = numProps + numEdits; size_t nBytes = 0;
  out.valBytesOff = end;
  if (nRec > 0) {
    patchByteLen.ensure(ctx, nRec + 1); patchByteOff.ensure(ctx, nRec + 2);
    foreach(ctx, nRec, PatchBytesCountKernel{propOut.p, numProps, editOut.p, patchByteLen.p});
    scan_exclusive(ctx, scanTmp, patchByteLen.p, patchByteOff.p, nRec);
    nBytes = readU32(patchByteOff.p + nRec);
    if ((u64)end + nBytes >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: patch larger than 4 GiB");
    patchBytesD.ensure(ctx, nBytes + 8);
    foreach(ctx, nRec, PatchBytesGatherKernel{arena.p, propOut.p, numProps, editOut.p, patchByteOff.p, (u32)out.valBytesOff, patchBytesD.p, errWord.p});
    if (const u64 ew = fetchErr()) throwPatchValueError(ew, numProps);
  }
  out.valBytesLen = nBytes; out.bigEnd = (out.valBytesOff + nBytes + 7) & ~(size_t)7;
  patchBuf.ensure(out.bigEnd + 4096);
  // the copy-out runs on the side stream: the caller joins it before reading the patch, later kernels overlap it
  side_fork(ctx);
  d2h_side(ctx, patchBuf.p + out.propsOff, propOut.p, numProps * sizeof(PropRec));
  if (numEdits > 0) { d2h_side(ctx, patchBuf.p + out.editsOff, editOut.p, numEdits * sizeof(EditRec)); if (shipElem) d2h_side(ctx, patchBuf.p + out.elemOff, editElem.p, numEdits * 8); }
  if (nBytes > 0) d2h_side(ctx, patchBuf.p + out.valBytesOff, patchBytesD.p, nBytes);
}

// a value that the reference's decodeValue refuses (it decodes every value that reaches a patch, columnar.js:300-329)
inline void Engine::throwPatchValueError(u64 ew, size_t numProps) {
  if ((ew & 0xff) == KE_FLOAT_LEN) { u32 l = 0; d2h(ctx, &l, patchByteLen.p + (ew >> 8), 4); sync(ctx); const size_t i = (size_t)(ew >> 8); u32 keyLen = 0; if (i < numProps) { PropRec r; d2h(ctx, &r, propOut.p + i, sizeof(PropRec)); sync(ctx); keyLen = r.keyLen == 0xffffffffu ? 0 : r.keyLen; } throw Error(AMG_ERR_RANGE, "Invalid length for floating point number: " + std::to_string(l - keyLen)); }
  throwKernelError(ew);
}

inline void Engine::getPatch(PatchOut& out) {
  clearErr();
  succCnt.ensure(ctx, numRows + 2);
  foreach(ctx, numRows, SuccCntFromOffKernel{succOff.p, succCnt.p});
  struct SideJoin { Ctx& c; ~SideJoin() { side_join(c); } } sideJoin{ctx};
  buildPatch(PatchInputs{doc.view(), numRows, true, succOff.p, succ.p, succCnt.p, Ord{actorRank.p, bits_for(std::max<size_t>(st.actorIds.size(), 2) - 1)}}, out);
  side_join(ctx); sync(ctx);
  checkErr();
  fillPatchHeader(out);
  finishPatch(out);
}


inline RawRows Engine::rawRows() {
  return RawRows{r_objActor.p, r_objCtr.p, r_keyActor.p, r_keyCtr.p, r_keyStrOff.p, r_keyStrLen.p, r_insert.p, r_action.p, r_valLen.p, r_valOff.p, r_predNum.p, r_predOff.p, r_predActor.p, r_predCtr.p};
}
// Fused header parse + column expansion of B changes (chOff / chLen are on the device). The raw row tables are sized from
// what earlier calls needed (else from the batch size); the kernel never writes outside them and reports an overflow.
inline DecodeTilesArgs Engine::decodeArgs(const u8* arenaP, size_t B, size_t batchBytes) {
  hot.ensure(ctx, B + 1); nOps.ensure(ctx, B + 1); nPreds.ensure(ctx, B + 1); nDeps.ensure(ctx, B + 1); nActors.ensure(ctx, B + 1);
  rawBase.ensure(ctx, B + 2); rawPredBase.ensure(ctx, B + 2); decErr.ensure(ctx, B + 1);
  decCursor.ensure(ctx, 8); decDirect.ensure(ctx, B + 2);   // decCursor: one 64-byte block = cursor (2 x u64), totals (4 x u32), direct count, done count
  const size_t wantRows = std::max(decWantRows, B + B / 4 + batchBytes / 256 + 1024), wantPreds = std::max(decWantPreds, B + B / 4 + batchBytes / 256 + 1024);
  for (DBuf<u32>* b : {&r_objActor, &r_objCtr, &r_keyActor, &r_keyCtr, &r_keyStrOff, &r_keyStrLen, &r_insert, &r_action, &r_valLen, &r_valOff, &r_predNum, &r_predOff}) b->ensure(ctx, wantRows + 1);
  r_predActor.ensure(ctx, wantPreds + 1); r_predCtr.ensure(ctx, wantPreds + 1);
  decRowCap = wantRows; decPredCap = wantPreds;
  return DecodeTilesArgs{arenaP, chOff.p, chLen.p, (u32)B, 0u, hot.p, nOps.p, nPreds.p, nDeps.p, nActors.p, rawBase.p, rawPredBase.p, decErr.p, rawRows(), (u32)wantRows, (u32)wantPreds,
                         (unsigned long long*)decCursor.p, decTotalsPtr(), errWord.p, 0u, decDirect.p, decTotalsPtr() + 4};
}
// the whole batch in one go (bytes resident): the range launch, the list launch over the inflated changes (numDefl of them,
// bytes from arena offset deflStart on), then the changes outside their tile's window
inline void Engine::runDecodeTiles(const u8* arenaP, size_t B, size_t batchBytes, const u32* deflListP, size_t numDefl, size_t deflStart) {
  DecodeTilesArgs a = decodeArgs(arenaP, B, batchBytes);
  if (numDefl > 0) a.skipFrom = (u32)deflStart;
  decode_tiles_begin(ctx, a); decode_tiles_range(ctx, a, 0, (u32)B);
  if (numDefl > 0) decode_tiles_list(ctx, a, deflListP, (u32)numDefl);
  decode_tiles_finish(ctx, a, B);
}
inline bool Engine::decodeOverflowed(const u32 totals[4]) {
  if (!totals[2]) return false;
  if (totals[0] >= (1u << 29)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^29 operations in one call");
  if (totals[1] >= (1u << 30)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^30 predecessors in one call");
  decWantRows = (size_t)totals[0] + 1024; decWantPreds = (size_t)totals[1] + 1024;
  return true;
}

// Values of columns with unknown ids in the changes this call applies (reference new.js:1406-1424 keeps them in the document).
// Host work on a rare path: headers, op counts and actor maps come back from the device, the change bytes from the arena.
inline void Engine::collectUnknownColumns(size_t B, std::vector<std::pair<u64, UnknownRow>>& out, std::set<u32>& ids) {
  std::vector<ChangeHot> hh(B); std::vector<u32> nops(B), amb(B + 1), nact(B); std::vector<u8> ap(B);
  d2h(ctx, hh.data(), hot.p, B * sizeof(ChangeHot)); d2h(ctx, nops.data(), nOps.p, B * 4); d2h(ctx, amb.data(), amapBase.p, (B + 1) * 4); d2h(ctx, nact.data(), nActors.p, B * 4); d2h(ctx, ap.data(), applied.p, B); sync(ctx);
  std::vector<u32> am(amb[B] + 1); if (amb[B]) { d2h(ctx, am.data(), amap.p, (size_t)amb[B] * 4); sync(ctx); }
  for (size_t b = 0; b < B; b++) {
    if (!ap[b] || nops[b] == 0 || hh[b].dataOff <= hh[b].dirOff) continue;
    const ChangeHot& h = hh[b];
    std::vector<u8> bytes(h.len); d2h(ctx, bytes.data(), arena.p + h.off, h.len); sync(ctx);
    std::vector<std::array<u32, 3>> cols; bool any = false;
    { ByteReader d(bytes.data(), h.dirOff - h.off, h.dataOff - h.off); u32 pos = h.dataOff - h.off;
      while (!d.done() && !d.err) { const u32 id = (u32)d.uleb(), l = (u32)d.uleb(); cols.push_back({id, pos, l}); if (!is_known_change_column(id)) any = true; pos += l; } }
    if (!any) continue;
    const u32 author = am[amb[b]];
    const u32 e = read_unknown_columns(bytes.data(), cols, nops[b], is_known_change_column, [&](size_t i, UnknownRow& row) {
      for (auto& kv : row) {
        ids.insert(kv.first);
        if ((kv.first & 7) == 1) for (auto& v : kv.second) if (!v.isNull) {   // ACTOR_ID: change-local index -> document actor index (new.js:586-588)
          if ((u64)v.num >= nact[b]) throw Error(AMG_ERR_RANGE, "actor index out of range");
          v.num = am[amb[b] + (u32)v.num];
        }
      }
      out.emplace_back(pack_id(h.startOp + i, author), row);
    });
    if (e == KE_UNSUPPORTED_OP) throw Error(AMG_ERR_RANGE, "unexpected VALUE_RAW column");
    if (e) throwKernelError(((u64)b << 8) | e);
  }
}

// save(): document columns of the unknown ids, rows in document order; a row without a value in a column contributes null
// (a group cardinality of 0 for grouped columns), as the reference's decoders yield for columns a block never had
// (new.js:1418-1420 makeDecoders over the widened column list).
inline void Engine::appendUnknownDocColumns(std::vector<std::pair<u32, std::string>>& cols) {
  const size_t N = numRows; std::vector<u64> ids(N); d2h(ctx, ids.data(), doc.id.p, N * 8); sync(ctx);
  for (u32 id : unknownCols.colIds) {
    std::vector<UnknownValue> vals; vals.reserve(N);
    const bool grouped = (id & 7) != 0 && (unknownCols.colIds.count((id & ~15u)) != 0 || (id >> 4) == 7 || (id >> 4) == 8);   // a member of a group with a GROUP_CARD column: a row without values has cardinality 0
    for (size_t i = 0; i < N; i++) {
      auto it = unknownCols.byOp.find(ids[i]);
      const std::vector<UnknownValue>* v = nullptr;
      if (it != unknownCols.byOp.end()) { auto c = it->second.find(id); if (c != it->second.end()) v = &c->second; }
      if (v) vals.insert(vals.end(), v->begin(), v->end());
      else if ((id & 7) == 0) { UnknownValue z; z.isNull = false; z.num = 0; vals.push_back(z); }   // GROUP_CARD: `readValue() || 0` (new.js:581)
      else if (!grouped && (id & 7) != 7) vals.push_back(UnknownValue());   // null (raw bytes: nothing)
    }
    cols.emplace_back(id, encode_unknown_column(id, vals));
  }
}

// Columns of bulk changes (>= HUGE_CHANGE_OPS ops) through the parallel column decoders. largeList holds the large changes of
// the batch (at most 8 here). hugeDone[k * NCOLS + col] = 1 tells DecodeColumnKernel that column `col` of large change k is done.
inline void Engine::decodeHugeChanges(const RawRows& raw, size_t numLarge) {
  static const u32 HUGE_CHANGE_OPS = 4096;
  hugeDone.ensure(ctx, numLarge * NCOLS + 1); dev_memset(ctx, hugeDone.p, 0, (numLarge * NCOLS + 1) * 4);
  std::vector<u32> list(numLarge); d2h(ctx, list.data(), largeList.p, numLarge * 4); sync(ctx);
  u32 any = 0;
  for (size_t k = 0; k < numLarge; k++) {
    const u32 c = list[k]; ChangeHot h; u32 n = 0, np = 0, rb = 0, rpb = 0;
    d2h(ctx, &h, hot.p + c, sizeof(ChangeHot)); d2h(ctx, &n, nOps.p + c, 4); d2h(ctx, &np, nPreds.p + c, 4); d2h(ctx, &rb, rawBase.p + c, 4); d2h(ctx, &rpb, rawPredBase.p + c, 4); sync(ctx);
    if (n < HUGE_CHANGE_OPS || h.dataOff <= h.dirOff || h.dataOff - h.dirOff > 4096) continue;
    std::vector<u8> dir(h.dataOff - h.dirOff); d2h(ctx, dir.data(), arena.p + h.dirOff, dir.size()); sync(ctx);
    u32 cOff[NCOLS] = {0}, cLen[NCOLS] = {0}; bool have[NCOLS] = {false};
    { ByteReader d(dir.data(), 0, (u32)dir.size()); u32 pos = h.dataOff;
      while (!d.done() && !d.err) { const u32 id = (u32)d.uleb(), l = (u32)d.uleb(); const int ix = col_index_of(id); if (ix >= 0) { cOff[ix] = pos; cLen[ix] = l; have[ix] = true; } pos += l; } }
    std::vector<u32> done(NCOLS, 0);
    for (int col = 0; col < NCOLS; col++) {
      const size_t cnt = (col == CX_PRED_ACTOR || col == CX_PRED_CTR) ? np : n;
      if (CX_PAR_KIND[col] == PK_NONE || !have[col] || cLen[col] == 0 || cnt == 0) continue;   // absent / empty: the serial path fills the defaults
      u64 sum = 0;
      bool ok = parCols.decode(CX_PAR_KIND[col], arena.p + cOff[col], cLen[col], cnt, cx_outputs(raw, col, rb, rpb, have[CX_VAL_RAW] ? cOff[CX_VAL_RAW] : 0, &sum));
      if (ok && col == CX_VAL_LEN) ok = sum <= (have[CX_VAL_RAW] ? cLen[CX_VAL_RAW] : 0);
      if (ok && col == CX_PRED_NUM) { ok = sum == np; if (ok && rpb) foreach(ctx, cnt, PcAddBaseKernel{raw.predOff + rb, rpb}); }
      if (ok) { done[col] = 1; any |= 1u << col; }
    }
    h2d(ctx, hugeDone.p + k * NCOLS, done.data(), NCOLS * 4); sync(ctx);
    if (trace.live) fprintf(stderr, "amgpu decode: bulk change %u (%u ops, %u preds): columns expanded in parallel: mask %04x\n", c, n, np, any);
  }
}

// Re-runs the decode kernels over the last applied batch (bytes resident in HBM) and times them with CUDA events.
// msParse = the fused decode (k_decode_tiles: header parse + expansion of every change of up to SMALL_CHANGE_OPS ops),
// msDec = DecodeColumnKernel over the larger changes (0 when the batch has none).
inline void Engine::benchDecode(int iters, float* msSha, float* msParse, float* msDec, u64* algoBytes) {
  if (lastB == 0 || iters <= 0) throw Error(AMG_ERR_RANGE, "amg_bench_decode: no batch has been applied yet");
  const size_t B = lastB;
  hashTmp.ensure(ctx, B * 32 + 64);
  RawRows raw = rawRows();
  *algoBytes = (u64)lastBytes + 48ull * lastM + 8ull * lastP + 96ull * B;
#ifndef AMG_EMU
  cudaEvent_t e[4]; for (auto& x : e) cudaEventCreate(&x);
  const u8* batchArena = arena.p;
  cudaEventRecord(e[0], ctx.stream);
  for (int i = 0; i < iters; i++) sha_range(ctx, ShaTilesArgs{batchArena, chOff.p, chLen.p, hashTmp.p, errWord.p, nullptr, 0u, (u32)B}, false);
  cudaEventRecord(e[1], ctx.stream);
  for (int i = 0; i < iters; i++) runDecodeTiles(batchArena, B, lastBytes, deflList.p, lastDeflCount, lastDeflStart);
  cudaEventRecord(e[2], ctx.stream);
  for (int i = 0; i < iters; i++) {
    if (lastNumLarge > 0) foreach(ctx, (size_t)NCOLS * lastNumLarge, DecodeColumnKernel{batchArena, largeList.p, lastNumLarge, hot.p, nOps.p, nPreds.p, rawBase.p, rawPredBase.p, applied.p, raw, errWord.p, nullptr});
  }
  cudaEventRecord(e[3], ctx.stream);
  CUDA_CHECK(cudaEventSynchronize(e[3]));
  float a, b, c; cudaEventElapsedTime(&a, e[0], e[1]); cudaEventElapsedTime(&b, e[1], e[2]); cudaEventElapsedTime(&c, e[2], e[3]);
  *msSha = a / iters; *msParse = b / iters; *msDec = lastNumLarge > 0 ? c / iters : 0.f;
  for (auto& x : e) cudaEventDestroy(x);
#else
  *msSha = *msParse = *msDec = 0;
#endif
}

// Change history of a loaded document (reference new.js:1887-1912 computeHashGraph -> columnar.js:876-981): rebuilds every
// loaded change - ops from the document rows and the deletions implied by their succ lists, preds, actor tables, canonical
// column bytes - and its hash. Kernels: history.cuh. Nothing persistent is touched until the heads check has passed.
inline void Engine::computeHashGraph() {
  if (loaded.haveHashGraph) return;
  if (!unknownCols.empty()) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: the change history of a loaded document that holds columns with unknown ids cannot be reconstructed");
  const size_t L = loaded.numChanges;
  if (L == 0) { loaded.haveHashGraph = true; return; }
  if (L >= (1u << 29) || numRows + numSucc >= (1u << 30)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: document too large for history reconstruction");
  HistoryCall h{L, numRows, numSucc, st.actorIds.size(), doc.view()};
  clearErr();
  histChangeColumns(h); histActorOrder(h); histPredsAndDeletions(h); histOpsToChanges(h); histActorTables(h);
  histEncode(h); histHashes(h); histCheckHeads(h); histCommit(h);
}

// Change metadata column k of the loaded document, `count` values: the parallel decoder when the history is long (it
// declines what is not canonical), else LoadedColKernel.
inline void Engine::decodeLoadedCol(int k, size_t count, long long* out, u32* strOff, u32* strLen) {
  const HostChange& c = loaded.cols[k]; const u32 rawOff = loaded.cols[CC_EXTRA_RAW].off;
  if (count >= parDocMinRows && c.len > 0 && parCols.decode(CHANGE_COLS[k].pk, arena.p + c.off, c.len, count, PcOut{nullptr, out, strOff, strLen, rawOff})) return;
  foreach_warp(ctx, 1, LoadedColKernel{CHANGE_COLS[k].lc, arena.p, c.off, c.len, rawOff, (u32)count, out, strOff, strLen, nullptr});
}

// 1. change metadata columns (the same decoders as save() after load())
inline void Engine::histChangeColumns(HistoryCall& h) {
  const size_t L = h.L;
  for (DBuf<long long>* b : {&h.cActor, &h.cSeq, &h.cMaxOp, &h.cTime, &h.cDepsNum, &h.cExtra, &h.scratchV}) b->ensure(ctx, L + 1);
  for (DBuf<u32>* b : {&h.msgOff, &h.msgLen, &h.extraOff, &h.extraLen, &h.tmpOff, &h.tmpLen, &h.depsNum32}) b->ensure(ctx, L + 2);
  h.depBase.ensure(ctx, L + 2);
  decodeLoadedCol(CC_ACTOR, L, h.cActor.p, h.tmpOff.p, h.tmpLen.p);
  decodeLoadedCol(CC_SEQ, L, h.cSeq.p, h.tmpOff.p, h.tmpLen.p);
  decodeLoadedCol(CC_MAX_OP, L, h.cMaxOp.p, h.tmpOff.p, h.tmpLen.p);
  decodeLoadedCol(CC_TIME, L, h.cTime.p, h.tmpOff.p, h.tmpLen.p);
  decodeLoadedCol(CC_MESSAGE, L, h.scratchV.p, h.msgOff.p, h.msgLen.p);
  decodeLoadedCol(CC_DEPS_NUM, L, h.cDepsNum.p, h.tmpOff.p, h.tmpLen.p);
  decodeLoadedCol(CC_EXTRA_LEN, L, h.cExtra.p, h.extraOff.p, h.extraLen.p);
  foreach(ctx, L, HistI64ToU32Kernel{h.cDepsNum.p, h.depsNum32.p});
  scan_exclusive(ctx, scanTmp, h.depsNum32.p, h.depBase.p, L);
  const size_t D = h.D = readU32(h.depBase.p + L);
  h.depIdxV.ensure(ctx, D + 1); h.depIdx.ensure(ctx, D + 2);
  if (D) { decodeLoadedCol(CC_DEPS_INDEX, D, h.depIdxV.p, h.tmpOff.p, h.tmpLen.p); foreach(ctx, D, HistI64ToU32Kernel{h.depIdxV.p, h.depIdx.p}); }
}

// 2. actor order (hex string order = byte order), representatives
inline void Engine::histActorOrder(HistoryCall& h) {
  const size_t A = h.A;
  std::vector<u32> order(A), rankH(A), repOffH(A), repLenH(A);
  for (size_t a = 0; a < A; a++) { order[a] = (u32)a; repOffH[a] = st.actorRep[a].first; repLenH[a] = st.actorRep[a].second; }
  std::sort(order.begin(), order.end(), [&](u32 x, u32 y) { return st.actorIds[x] < st.actorIds[y]; });
  for (size_t i = 0; i < A; i++) rankH[order[i]] = (u32)i;
  for (DBuf<u32>* b : {&h.rankD, &h.actorOfRank, &h.repOff, &h.repLen}) b->ensure(ctx, A + 1);
  h2d(ctx, h.rankD.p, rankH.data(), A * 4); h2d(ctx, h.actorOfRank.p, order.data(), A * 4); h2d(ctx, h.repOff.p, repOffH.data(), A * 4); h2d(ctx, h.repLen.p, repLenH.data(), A * 4);
  h.ctrBits = bits_for(st.maxOp + 1); h.idBits = std::min(64, h.ctrBits + 16);
  trace.print("history", "change columns decoded", h.t0);
}

// 3. (successor, predecessor) pairs -> pred lists and deletions
inline void Engine::histPredsAndDeletions(HistoryCall& h) {
  const size_t N = h.N, S = h.S;
  h.idSorted.ensure(ctx, N + 1); h.idRows.ensure(ctx, N + 1);
  if (N) { foreach(ctx, N, HistIdKeyKernel{h.d, h.idSorted.p, h.idRows.p}); radix_sort_pairs(ctx, sortTmp, h.idSorted, h.idRows, N, 0, h.idBits); }
  for (DBuf<u64>* b : {&h.predKey, &h.succKey, &h.keyA, &h.keyB}) b->ensure(ctx, S + 1);
  for (DBuf<u32>* b : {&h.pairRow, &h.valA, &h.pairRowSorted, &h.head, &h.groupIdx}) b->ensure(ctx, S + 2);
  if (S) {
    foreach(ctx, N, HistPairKernel{h.d, succOff.p, succ.p, h.rankD.p, h.predKey.p, h.succKey.p, h.pairRow.p});
    foreach(ctx, S, HistIotaKernel{h.valA.p});
    d2d(ctx, h.keyA.p, h.predKey.p, S * 8);
    radix_sort_pairs(ctx, sortTmp, h.keyA, h.valA, S, 0, h.idBits);                 // by predecessor (counter, actor order) ...
    foreach(ctx, S, HistGatherKeyKernel{h.succKey.p, h.valA.p, h.keyB.p});
    radix_sort_pairs(ctx, sortTmp, h.keyB, h.valA, S, 0, h.idBits);                 // ... then, stably, by successor id
    foreach(ctx, S, HistGatherU32Kernel{h.pairRow.p, h.valA.p, h.pairRowSorted.p});
    foreach(ctx, S, HistGroupHeadKernel{h.keyB.p, h.head.p});
    scan_exclusive(ctx, scanTmp, h.head.p, h.groupIdx.p, S);
    h.G = readU32(h.groupIdx.p + S);
  }
  const size_t G = h.G;
  for (DBuf<u32>* b : {&h.groupStart, &h.groupRow, &h.isDel, &h.delSlot}) b->ensure(ctx, G + 2);
  h.groupId.ensure(ctx, G + 1);
  if (G) {
    foreach(ctx, S, HistGroupKernel{h.head.p, h.groupIdx.p, h.keyB.p, (u32)S, h.idSorted.p, h.idRows.p, (u32)N, h.groupStart.p, h.groupId.p, h.groupRow.p, h.isDel.p});
    scan_exclusive(ctx, scanTmp, h.isDel.p, h.delSlot.p, G);
    h.numDel = readU32(h.delSlot.p + G);
  }
  const size_t M = h.M = N + h.numDel;
  h.opId.ensure(ctx, M + 1); for (DBuf<u32>* b : {&h.opSrc, &h.opPredStart, &h.opPredNum, &h.opOrder, &h.opChange, &h.predNumSorted}) b->ensure(ctx, M + 2);
  h.opPredBase.ensure(ctx, M + 3);
  if (N) foreach(ctx, N, HistRowOpKernel{h.d, h.opId.p, h.opSrc.p, h.opPredStart.p, h.opPredNum.p});
  if (G) foreach(ctx, G, HistGroupOpKernel{h.groupStart.p, h.groupId.p, h.groupRow.p, h.isDel.p, h.delSlot.p, h.pairRowSorted.p, (u32)G, (u32)S, (u32)N, h.opId.p, h.opSrc.p, h.opPredStart.p, h.opPredNum.p});
  trace.print("history", "preds and deletions", h.t0);
}

// 4. ops by (actor, counter); changes by (actor, seq); every op finds its change
inline void Engine::histOpsToChanges(HistoryCall& h) {
  const size_t L = h.L, A = h.A, M = h.M;
  h.opKey.ensure(ctx, M + 1); h.chKey.ensure(ctx, L + 1);
  h.changeOrder.ensure(ctx, L + 1); h.actorStart.ensure(ctx, A + 2); h.chOpStart.ensure(ctx, L + 2); h.chNOps.ensure(ctx, L + 2);
  if (M) { foreach(ctx, M, HistOpKeyKernel{h.opId.p, h.opKey.p, h.opOrder.p}); radix_sort_pairs(ctx, sortTmp, h.opKey, h.opOrder, M, 0, h.ctrBits); radix_sort_pairs(ctx, sortTmp, h.opKey, h.opOrder, M, 48, 64); }
  foreach(ctx, L, HistChangeKeyKernel{h.cActor.p, h.cSeq.p, h.chKey.p, h.changeOrder.p});
  radix_sort_pairs(ctx, sortTmp, h.chKey, h.changeOrder, L, 0, 40); radix_sort_pairs(ctx, sortTmp, h.chKey, h.changeOrder, L, 40, 57);
  foreach(ctx, A + 1, HistLowerBoundKernel{h.chKey.p, (u32)L, 40, h.actorStart.p});
  dev_memset(ctx, h.chOpStart.p, 0, (L + 1) * 4); dev_memset(ctx, h.chNOps.p, 0, (L + 1) * 4);
  if (M) {
    foreach(ctx, M, HistAssignKernel{h.opKey.p, h.actorStart.p, h.changeOrder.p, h.cMaxOp.p, (u32)A, numApplied == L ? 1 : 0, h.opChange.p, errWord.p});
    foreach(ctx, M, HistChangeStartKernel{h.opChange.p, h.chOpStart.p});
    foreach(ctx, M, HistChangeCountKernel{h.opChange.p, h.chNOps.p});
    foreach(ctx, M, HistCheckIdsKernel{h.opKey.p, h.opChange.p, h.chOpStart.p, h.chNOps.p, h.cMaxOp.p, errWord.p});
    foreach(ctx, M, HistPredNumSortedKernel{h.opPredNum.p, h.opOrder.p, h.predNumSorted.p});
    scan_exclusive(ctx, scanTmp, h.predNumSorted.p, h.opPredBase.p, M);
  } else dev_memset(ctx, h.opPredBase.p, 0, 8);
  h.P = M ? readU32(h.opPredBase.p + M) : 0;
  checkErr();
  trace.print("history", "ops assigned to changes", h.t0);
}

// 5. the other actors of every change
inline void Engine::histActorTables(HistoryCall& h) {
  const size_t L = h.L, M = h.M; const HistOpView view = h.view();
  h.slotCnt.ensure(ctx, M + 2); h.slotBase.ensure(ctx, M + 3); h.otherStart.ensure(ctx, L + 3);
  if (M) { foreach(ctx, M, HistActorSlotCountKernel{view, h.slotCnt.p}); scan_exclusive(ctx, scanTmp, h.slotCnt.p, h.slotBase.p, M); h.Q = readU32(h.slotBase.p + M); }
  const size_t Q = h.Q;
  h.slotKey.ensure(ctx, Q + 1); h.slotVal.ensure(ctx, Q + 1); h.uniq.ensure(ctx, Q + 2); h.uniqSlot.ensure(ctx, Q + 3);
  if (Q) {
    foreach(ctx, M, HistActorPairKernel{view, h.slotBase.p, h.opChange.p, h.cActor.p, h.rankD.p, h.slotKey.p});
    foreach(ctx, Q, HistIotaKernel{h.slotVal.p});
    radix_sort_pairs(ctx, sortTmp, h.slotKey, h.slotVal, Q, 0, 64);
    foreach(ctx, Q, HistUniqueKernel{h.slotKey.p, h.uniq.p});
    scan_exclusive(ctx, scanTmp, h.uniq.p, h.uniqSlot.p, Q);
    h.U = readU32(h.uniqSlot.p + Q);
  }
  h.other.ensure(ctx, h.U + 1);
  if (h.U) foreach(ctx, Q, HistOtherFillKernel{h.slotKey.p, h.uniq.p, h.uniqSlot.p, h.other.p});
  foreach(ctx, L + 1, HistLowerBoundKernel{h.other.p, (u32)h.U, 16, h.otherStart.p});
  trace.print("history", "actor tables", h.t0);
}

// 6. local actor indexes and delta values, then the bytes (two passes)
inline void Engine::histEncode(HistoryCall& h) {
  const size_t L = h.L, M = h.M, P = h.P; const HistOpView view = h.view();
  h.objA.ensure(ctx, M + 1); h.keyAi.ensure(ctx, M + 1); h.keyDelta.ensure(ctx, M + 1); h.predA.ensure(ctx, P + 1); h.predDelta.ensure(ctx, P + 1);
  for (DBuf<u32>* b : {&h.outLen, &h.depsAt, &h.bodyAt, &h.chOffD}) b->ensure(ctx, L + 2);
  h.outOff.ensure(ctx, L + 3);
  HistChanges hc{h.cActor.p, h.cSeq.p, h.cMaxOp.p, h.cTime.p, h.msgOff.p, h.msgLen.p, h.cDepsNum.p, h.extraOff.p, h.extraLen.p};
  foreach(ctx, L, HistPrepKernel{view, hc, h.chOpStart.p, h.chNOps.p, h.opPredBase.p, h.other.p, h.otherStart.p, h.rankD.p, h.objA.p, h.keyAi.p, h.keyDelta.p, h.predA.p, h.predDelta.p});
  HistEncodeKernel enc{0, view, hc, arena.p, h.chOpStart.p, h.chNOps.p, h.opPredBase.p, (u32)M, (u32)P, h.other.p, h.otherStart.p, h.repOff.p, h.repLen.p, h.actorOfRank.p,
                       h.objA.p, h.keyAi.p, h.keyDelta.p, h.predA.p, h.predDelta.p, h.outLen.p, h.outOff.p, nullptr, 0, h.depsAt.p, h.bodyAt.p};
  foreach(ctx, L, enc);
  scan_exclusive(ctx, scanTmp, h.outLen.p, h.outOff.p, L);
  excl64.ensure(ctx, L + 2); scan_exclusive64(ctx, scanTmp, ParColumnDecoder::PcDeltaInputU32{h.outLen.p}, excl64.p, L);
  u64 tot64 = 0; u32 lastLen = 0; d2h(ctx, &tot64, excl64.p + L - 1, 8); d2h(ctx, &lastLen, h.outLen.p + L - 1, 4); sync(ctx);
  const u64 T = h.T = tot64 + lastLen;
  if ((u64)arenaLen + T + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per document");
  arena.ensure(ctx, arenaLen + T + 64, arenaLen);
  enc.pass = 1; enc.arena = arena.p; enc.outArena = arena.p; enc.outBase = (u32)arenaLen;
  foreach(ctx, L, enc);
  foreach(ctx, L, HistChOffKernel{h.outOff.p, (u32)arenaLen, h.chOffD.p});
  checkErr();
  trace.print("history", "changes encoded", h.t0);
}

// 7. dependency levels (host: one pass over the dependency indexes), hashes level by level
inline void Engine::histHashes(HistoryCall& h) {
  const size_t L = h.L, D = h.D;
  std::vector<u32> depsNumH(L), depBaseH(L + 1), depIdxH(D), level(L), list(L);
  d2h(ctx, depsNumH.data(), h.depsNum32.p, L * 4); d2h(ctx, depBaseH.data(), h.depBase.p, (L + 1) * 4); if (D) d2h(ctx, depIdxH.data(), h.depIdx.p, D * 4); sync(ctx);
  u32 maxLevel = 0; h.isDep.assign(L, 0);
  for (size_t k = 0; k < L; k++) {
    u32 lv = 0;
    for (u32 i = 0; i < depsNumH[k]; i++) { const u32 di = depIdxH[depBaseH[k] + i]; if (di >= k) throw Error(AMG_ERR_RANGE, "No hash for index " + std::to_string(di) + " while processing index " + std::to_string(k)); lv = std::max(lv, level[di] + 1); h.isDep[di] = 1; }
    level[k] = lv; maxLevel = std::max(maxLevel, lv);
  }
  std::vector<u32> levelStart(maxLevel + 2, 0);
  for (size_t k = 0; k < L; k++) levelStart[level[k] + 1]++;
  for (u32 l = 0; l <= maxLevel; l++) levelStart[l + 1] += levelStart[l];
  { std::vector<u32> at(levelStart.begin(), levelStart.end() - 1); for (size_t k = 0; k < L; k++) list[at[level[k]]++] = (u32)k; }
  h.listD.ensure(ctx, L + 1); h2d(ctx, h.listD.p, list.data(), L * 4);
  h.newHashes.ensure(ctx, L * 32 + 64); d2d(ctx, h.newHashes.p, hashes.p, L * 32);   // scratch copy: committed only after the heads check
  const HistHashKernel hk{h.listD.p, arena.p, h.chOffD.p, h.outLen.p, h.depsAt.p, h.bodyAt.p, h.cDepsNum.p, h.depBase.p, h.depIdx.p, (u32)L, h.newHashes.p, errWord.p};
  auto wide = [&](u32 l) { HistHashKernel k = hk; k.list = h.listD.p + levelStart[l]; const size_t cnt = levelStart[l + 1] - levelStart[l]; if (cnt) foreach(ctx, cnt, k); };
#ifdef AMG_EMU
  for (u32 l = 0; l <= maxLevel; l++) wide(l);
#else
  {
    DBuf<u32> levelStartD; levelStartD.ensure(ctx, levelStart.size() + 1); h2d(ctx, levelStartD.p, levelStart.data(), levelStart.size() * 4);
    const u32 kNarrow = 1024;   // levels up to this many changes are walked by one CTA (k_hist_hash_chain); wider ones get their own launch
    for (u32 l = 0; l <= maxLevel;) {
      if (levelStart[l + 1] - levelStart[l] > kNarrow) { wide(l); l++; continue; }
      u32 r = l; while (r <= maxLevel && levelStart[r + 1] - levelStart[r] <= kNarrow) r++;
      k_hist_hash_chain<<<1, 256, 0, ctx.stream>>>(hk, levelStartD.p, l, r - l);
      CUDA_CHECK(cudaGetLastError()); ctx.launches++;
      l = r;
    }
    sync(ctx);   // levelStartD is a local
  }
#endif
  checkErr();
  trace.print("history", "hashes (all levels)", h.t0);
}

// 8. heads: the changes nobody depends on must be exactly the document's heads (columnar.js:968-980)
inline void Engine::histCheckHeads(HistoryCall& h) {
  const size_t L = h.L;
  size_t nHeads = 0; for (size_t k = 0; k < L; k++) if (!h.isDep[k]) nHeads++;
  bool ok = numApplied != L || nHeads == st.heads.size();   // (changes applied after the load have moved the heads)
  std::vector<std::array<u8, 32>> got(st.heads.size());
  if (loaded.headIndexesUnknown) {   // loaded without head indexes: the heads are the changes nobody depends on, matched by hash
    if (numApplied != L) throw Error(AMG_ERR_INTERNAL, "amgpu: head indexes must be resolved right after the load");
    std::vector<u32> cand; for (size_t k = 0; k < L; k++) if (!h.isDep[k]) cand.push_back((u32)k);
    ok = cand.size() == st.heads.size();
    std::vector<std::array<u8, 32>> ch(cand.size());
    if (ok) { for (size_t i = 0; i < cand.size(); i++) d2h(ctx, ch[i].data(), h.newHashes.p + (size_t)cand[i] * 32, 32); sync(ctx); }
    for (size_t i = 0; i < st.heads.size() && ok; i++) {
      size_t j = 0; while (j < cand.size() && ch[j] != st.heads[i]) j++;
      if (j == cand.size()) ok = false; else st.headIdx[i] = cand[j];
    }
    if (ok) loaded.headIndexesUnknown = false;
  } else if (numApplied == L) {
    for (size_t i = 0; i < st.heads.size(); i++) d2h(ctx, got[i].data(), h.newHashes.p + (size_t)st.headIdx[i] * 32, 32);
    sync(ctx);
    for (size_t i = 0; i < st.heads.size() && ok; i++) if (h.isDep[st.headIdx[i]] || got[i] != st.heads[i]) ok = false;
  }
  if (!ok) throw Error(AMG_ERR_RANGE, "Mismatched heads hashes: the document's heads are not the hashes of its reconstructed changes");
  trace.print("history", "heads checked", h.t0);
}

// 9. commit: bytes into the arena and its host mirror, hashes, change table
inline void Engine::histCommit(HistoryCall& h) {
  const size_t L = h.L; const u64 T = h.T;
  if (hostArena.size() == arenaLen) {   // the mirror is complete: keep it complete (otherwise it is fetched when asked for)
    hostArena.resize(arenaLen + T);
    if (T) d2h(ctx, hostArena.data() + arenaLen, arena.p + arenaLen, T);
  }
  d2d(ctx, hashes.p, h.newHashes.p, L * 32);
  std::vector<u32> offH(L), lenH(L); d2h(ctx, offH.data(), h.chOffD.p, L * 4); d2h(ctx, lenH.data(), h.outLen.p, L * 4); sync(ctx);
  for (size_t k = 0; k < L; k++) changes[k] = HostChange{offH[k], lenH[k]};
  arenaLen += T; loaded.haveHashGraph = true; loaded.historyRebuilt = L;
  trace.print("history", "committed", h.t0);
}

// Parity hook: one document column through the parallel or the serial decoder (include/amgpu.h)
inline int Engine::debugDecodeColumn(const u8* bytes, size_t len, int kind, size_t n, bool parallel, long long* out) {
  if (kind < 0 || kind > 3 || len >= 0x7fffffffULL || n >= 0x7fffffffULL) throw Error(AMG_ERR_RANGE, "amg_debug_decode_column: bad arguments");
  DBuf<u8> colBytes; DBuf<long long> outD; DBuf<u32> tmp;
  colBytes.ensure(ctx, len + 64); dev_memset(ctx, colBytes.p, 0, len + 64); if (len) h2d(ctx, colBytes.p, bytes, len);
  outD.ensure(ctx, n + 1); tmp.ensure(ctx, n + 1);
  if (parallel) {
    static const int PK[4] = {PK_UINT, PK_INT, PK_DELTA, PK_BOOL};   // kind 3 (boolean) decodes into u32 rows, widened below
    const bool ok = parCols.decode(PK[kind], colBytes.p, len, n, kind == 3 ? PcOut{tmp.p} : PcOut{nullptr, outD.p});
    if (!ok) { sync(ctx); return 1; }
    if (kind == 3 && n) foreach(ctx, n, U32ToI64Kernel{tmp.p, outD.p});
  } else {
    clearErr();
    foreach_warp(ctx, 1, DebugColumnKernel{kind, colBytes.p, (u32)len, (u32)n, outD.p, tmp.p, errWord.p});
    checkErr();
  }
  if (n) d2h(ctx, out, outD.p, n * 8);
  sync(ctx);
  return 0;
}

// Parity hook: hashes, op counts and the raw decoded columns (change-local values) of a batch, without touching the document.
inline void Engine::decodeRaw(const u8* blob, const u64* offsets, size_t n, u8* hashesOut, u32* nOpsOut, u32** rowsOut, size_t* totalOps, size_t* totalPreds) {
  std::vector<u32> off(n), len(n); std::string staged;
  for (size_t i = 0; i < n; i++) {
    const u8* p = blob + offsets[i]; const size_t l = offsets[i + 1] - offsets[i];
    std::string inflated; if (l > 8 && p[8] == 2) inflated = inflateChange(p, l);
    off[i] = (u32)staged.size(); len[i] = (u32)(inflated.empty() ? l : inflated.size());
    if (inflated.empty()) staged.append((const char*)p, l); else staged += inflated;
  }
  DBuf<u8> ar; ar.ensure(ctx, staged.size() + 64); h2d(ctx, ar.p, staged.data(), staged.size()); dev_memset(ctx, ar.p + staged.size(), 0, 64);
  chOff.ensure(ctx, n); chLen.ensure(ctx, n); h2d(ctx, chOff.p, off.data(), n * 4); h2d(ctx, chLen.p, len.data(), n * 4);
  clearErr(); hashTmp.ensure(ctx, n * 32 + 64);
  foreach(ctx, n, ShaKernel{ar.p, chOff.p, chLen.p, hashTmp.p, errWord.p, nullptr, nullptr});
  applied.ensure(ctx, n); dev_memset(ctx, applied.p, 1, n);
  u32 tot[4] = {0, 0, 0, 0}; void* dst[4] = {&tot[0], &tot[1], &tot[2], &tot[3]};
  runDecodeTiles(ar.p, n, staged.size());
  readWords({{decTotalsPtr(), 4}, {decTotalsPtr() + 1, 4}, {decTotalsPtr() + 2, 4}, {decTotalsPtr() + 3, 4}}, dst);
  if (decodeOverflowed(tot)) { runDecodeTiles(ar.p, n, staged.size()); readWords({{decTotalsPtr(), 4}, {decTotalsPtr() + 1, 4}, {decTotalsPtr() + 2, 4}, {decTotalsPtr() + 3, 4}}, dst); }
  checkErr();
  const size_t M = tot[0];
  RawRows raw = rawRows();
  if (tot[3] & 1u) {
    largeFlag.ensure(ctx, n + 1); largeSlot.ensure(ctx, n + 2); largeList.ensure(ctx, n + 1);
    foreach(ctx, n, LargeFlagKernel{nOps.p, applied.p, largeFlag.p});
    scan_exclusive(ctx, scanTmp, largeFlag.p, largeSlot.p, n);
    const size_t nl = readU32(largeSlot.p + n);
    if (nl > 0) {
      foreach(ctx, n, CompactKernel{largeFlag.p, largeSlot.p, largeList.p});
      foreach(ctx, (size_t)NCOLS * nl, DecodeColumnKernel{ar.p, largeList.p, nl, hot.p, nOps.p, nPreds.p, rawBase.p, rawPredBase.p, applied.p, raw, errWord.p, nullptr});
    }
  }
  foreach(ctx, n, RaiseDecErrKernel{decErr.p, errWord.p});
  checkErr();
  d2h(ctx, hashesOut, hashTmp.p, n * 32); d2h(ctx, nOpsOut, nOps.p, n * 4);
  const size_t P = tot[1];
  opBase.ensure(ctx, n + 1); predBase.ensure(ctx, n + 1);
  scan_exclusive(ctx, scanTmp, nOps.p, opBase.p, n); scan_exclusive(ctx, scanTmp, nPreds.p, predBase.p, n);
  DBuf<u32> gathered; gathered.ensure(ctx, 12 * (M + 1) + 2 * (P + 1));
  if (M) foreach(ctx, M, GatherRawKernel{n, opBase.p, predBase.p, rawBase.p, rawPredBase.p, raw, gathered.p, M, gathered.p + 12 * M, P});
  u32* rows = (u32*)malloc(sizeof(u32) * (12 * (M + 1) + 2 * (P + 1)));
  d2h(ctx, rows, gathered.p, (12 * M + 2 * P) * 4);
  if (totalPreds) *totalPreds = P;
  sync(ctx); *rowsOut = rows; *totalOps = M; lastB = 0;
}


extern "C" void amg_host_sha256(const uint8_t* data, size_t len, uint8_t out[32]);   // hostsha.cc (x86 SHA extensions when present)
inline void host_sha256(const u8* data, size_t len, u8 out[32]) { amg_host_sha256(data, len, out); }

// Backend.save() (reference new.js:2033-2055, columnar.js:983-1004): change metadata columns (re-derived from the change
// headers that live in the arena) and the 16 document op columns (from the document table and its succ lists), encoded
// on the device (encode.cuh); the container (column directory, DEFLATE of columns >= 256 bytes, checksum) is assembled
// on the host, as the reference does.
inline void Engine::saveDocument(std::string& result) {
  if (!loaded.bytes.empty()) { result = loaded.bytes; return; }   // unchanged since Backend.load (new.js:2034)
  if (!encoder) encoder.reset(new ColumnEncoder(ctx, scanTmp));
  encoder->outLen = 0;
  SaveCall s{numApplied, numRows, numSucc, loaded.numChanges, numApplied - loaded.numChanges};
  clearErr();
  saveVals.ensure(ctx, std::max(std::max(s.C, s.N), s.S) + 2);
  saveChangeColumns(s); saveOpColumns(s); packDocument(s, result);
}

// change metadata (new.js:1680-1692 appendChange); the first L rows come from the loaded document's own columns
inline void Engine::saveChangeColumns(SaveCall& s) {
  const size_t C = s.C, N = s.N, L = s.L;
  if (C == 0) return;
  ColumnEncoder& enc = *encoder;
  ChangeMetaCall m{C, L, s.K};
  parseChangeMeta(m);
  const u32 loadedDeps = m.loadedDeps, totalDeps = m.laterDeps;
  saveVals.ensure(ctx, std::max<size_t>(std::max(std::max(C, N), s.S), (size_t)loadedDeps + totalDeps) + 2);
  saveStrOff.ensure(ctx, std::max(C, N) + 1); saveStrLen.ensure(ctx, std::max(C, N) + 1);
  auto col = [&](int k) { changeMetaColumn(m, k, saveVals.p, saveStrOff.p, saveStrLen.p); };
  auto add = [&](int k, size_t len) { s.changeCols.push_back({CHANGE_COLS[k].id, enc.outLen - len, len}); };
  col(CC_ACTOR);      add(CC_ACTOR, enc.rleNum(saveVals.p, C, false));
  col(CC_SEQ);        add(CC_SEQ, enc.deltaNum(saveVals.p, C));
  col(CC_MAX_OP);     add(CC_MAX_OP, enc.deltaNum(saveVals.p, C));
  col(CC_TIME);       add(CC_TIME, enc.deltaNum(saveVals.p, C));
  col(CC_MESSAGE);    add(CC_MESSAGE, enc.rle(StrCol{arena.p, saveStrOff.p, saveStrLen.p}, C));
  col(CC_DEPS_NUM);   add(CC_DEPS_NUM, enc.rleNum(saveVals.p, C, false));
  col(CC_DEPS_INDEX); add(CC_DEPS_INDEX, enc.deltaNum(saveVals.p, (size_t)loadedDeps + totalDeps));
  col(CC_EXTRA_LEN);  add(CC_EXTRA_LEN, enc.rleNum(saveVals.p, C, false));
                      add(CC_EXTRA_RAW, enc.raw(arena.p, saveStrOff.p, saveStrLen.p, C));
  checkErr();
}

inline void Engine::parseChangeMeta(ChangeMetaCall& m) {
  const size_t C = m.C, L = m.L, K = m.K;
  if (K > 0) {
    m.laterDeps = parseChangeHeaders(arena.p, changes.data() + L, K);
    resolveChangeDeps(arena.p, hashes.p, C, K, L, m.laterDeps);
  }
  if (L > 0) {   // number of dependency indexes the loaded changes carry
    DBuf<u64>& sumD = pairSucc; sumD.ensure(ctx, 1);
    const HostChange& dn = loaded.cols[CC_DEPS_NUM];
    u64 sum = 0;
    if (!(L >= parDocMinRows && dn.len > 0 && parCols.sumColumn(arena.p + dn.off, dn.len, L, &sum))) {
      foreach_warp(ctx, 1, LoadedColKernel{LC_SUM, arena.p, dn.off, dn.len, 0, 0, nullptr, nullptr, nullptr, sumD.p});
      d2h(ctx, &sum, sumD.p, 8); sync(ctx);
    }
    m.loadedDeps = (u32)sum;
  }
}

// Dependency indexes of K changes: parseChangeHeaders parses the headers at `pairs` in `ar` into meta / nDeps / depBase and
// returns the number of dependency hashes; resolveChangeDeps looks them up among hashes [0, C) into depIdx and returns the
// table's mask. `base`: ResolveDepsKernelT's numApplied (with 0 only depIdx is meaningful). Neither checks the error word; a
// caller that checks it right after parseChangeHeaders gets it with the total, at no extra read.
inline u32 Engine::parseChangeHeaders(const u8* ar, const HostChange* pairs, size_t K) {
  chPairs.ensure(ctx, K); chOff.ensure(ctx, K); chLen.ensure(ctx, K);
  h2d(ctx, chPairs.p, pairs, K * sizeof(HostChange));
  foreach(ctx, K, SplitPairsKernel{chPairs.p, chOff.p, chLen.p});
  meta.ensure(ctx, K); colOff.ensure(ctx, (size_t)NCOLS * K); colLen.ensure(ctx, (size_t)NCOLS * K);
  nOps.ensure(ctx, K + 1); nPreds.ensure(ctx, K + 1); nDeps.ensure(ctx, K + 1); nActors.ensure(ctx, K + 1);
  foreach(ctx, K, ParseKernel{ar, chOff.p, chLen.p, K, meta.p, colOff.p, colLen.p, nOps.p, nPreds.p, nDeps.p, nActors.p, errWord.p, flagWord.p + 8});
  depBase.ensure(ctx, K + 1); scan_exclusive(ctx, scanTmp, nDeps.p, depBase.p, K);
  return readU32(depBase.p + K);
}

inline u64 Engine::resolveChangeDeps(const u8* ar, const u8* hs, size_t C, size_t K, size_t base, u32 totalDeps) {
  depIdx.ensure(ctx, (size_t)totalDeps + 1); primary.ensure(ctx, K);
  const u64 mask = hashTableOf(hs, C);
  foreach(ctx, K, ResolveDepsKernelT<ChangeMeta>{ar, hs, hashTable.p, mask, meta.p, nDeps.p, base, depBase.p, depIdx.p, primary.p});
  return mask;
}

inline void Engine::changeMetaColumn(const ChangeMetaCall& m, int col, long long* out, u32* strOff, u32* strLen) {
  const size_t L = m.L, K = m.K;
  if (col == CC_DEPS_INDEX) {
    if (L > 0) decodeLoadedCol(CC_DEPS_INDEX, m.loadedDeps, out, strOff, strLen);
    if (m.laterDeps > 0) foreach(ctx, m.laterDeps, SaveDepIndexKernel{depIdx.p, out + m.loadedDeps});
    return;
  }
  if (L > 0) decodeLoadedCol(col, L, out, strOff, strLen);
  if (K == 0) return;
  if (col == CC_MESSAGE) { foreach(ctx, K, SaveMessageKernel{meta.p, strOff + L, strLen + L}); return; }
  int which = SM_ACTOR;
  switch (col) {
    case CC_ACTOR: which = SM_ACTOR; break; case CC_SEQ: which = SM_SEQ; break; case CC_MAX_OP: which = SM_MAX_OP; break;
    case CC_TIME: which = SM_TIME; break; case CC_DEPS_NUM: which = SM_DEPS_NUM; break; case CC_EXTRA_LEN: which = SM_EXTRA_LEN; break;
    default: throw Error(AMG_ERR_INTERNAL, "changeMetaColumn: no values for column " + std::to_string(col));
  }
  foreach(ctx, K, SaveChangeValKernel{which, arena.p, meta.p, actorSlots.p, (u64)actorCap - 1, out + L, strOff + L, strLen + L, errWord.p});
}

// document ops (columnar.js:60-82); chldActor / chldCtr are always null in this format version: empty
inline void Engine::saveOpColumns(SaveCall& s) {
  const size_t N = s.N, S = s.S;
  ColumnEncoder& enc = *encoder;
  auto add = [&](int k, size_t len) { s.opCols.push_back({DOC_COL_IDS[k], enc.outLen - len, len}); };
  if (N > 0) {
    DocRows d = doc.view();
    saveStrOff.ensure(ctx, N + 1); saveStrLen.ensure(ctx, N + 1);
    auto opVal = [&](int which) { foreach(ctx, N, SaveOpValKernel{which, d, succOff.p, saveVals.p}); };
    opVal(SC_OBJ_ACTOR); add(OC_OBJ_ACTOR, enc.rleNum(saveVals.p, N, false));
    opVal(SC_OBJ_CTR);   add(OC_OBJ_CTR, enc.rleNum(saveVals.p, N, false));
    opVal(SC_KEY_ACTOR); add(OC_KEY_ACTOR, enc.rleNum(saveVals.p, N, false));
    opVal(SC_KEY_CTR);   add(OC_KEY_CTR, enc.deltaNum(saveVals.p, N));
                         add(OC_KEY_STR, enc.rle(StrCol{arena.p, d.keyStrOff, d.keyStrLen}, N));
    opVal(SC_ID_ACTOR);  add(OC_ID_ACTOR, enc.rleNum(saveVals.p, N, false));
    opVal(SC_ID_CTR);    add(OC_ID_CTR, enc.deltaNum(saveVals.p, N));
    foreach(ctx, N, SaveInsertKernel{d, saveStrLen.p});
                         add(OC_INSERT, enc.boolean(saveStrLen.p, N));
    opVal(SC_ACTION);    add(OC_ACTION, enc.rleNum(saveVals.p, N, false));
    opVal(SC_VAL_LEN);   add(OC_VAL_LEN, enc.rleNum(saveVals.p, N, false));
    foreach(ctx, N, SaveValBytesKernel{d, saveStrLen.p});
                         add(OC_VAL_RAW, enc.raw(arena.p, d.valOff, saveStrLen.p, N));
    opVal(SC_SUCC_NUM);  add(OC_SUCC_NUM, enc.rleNum(saveVals.p, N, false));
    if (S > 0) {
      foreach(ctx, S, SaveSuccValKernel{0, succ.p, saveVals.p}); add(OC_SUCC_ACTOR, enc.rleNum(saveVals.p, S, false));
      foreach(ctx, S, SaveSuccValKernel{1, succ.p, saveVals.p}); add(OC_SUCC_CTR, enc.deltaNum(saveVals.p, S));
    }
  }
  trace.print("save", "columns encoded (device)", s.t0);
}

// host: DEFLATE of large columns (columnar.js:1052-1057), directory, container (columnar.js:659-686)
inline void Engine::packDocument(SaveCall& s, std::string& result) {
  const ColumnEncoder& enc = *encoder;
  std::vector<u8> raw(enc.outLen);
  if (enc.outLen) { d2h(ctx, raw.data(), enc.out.p, enc.outLen); sync(ctx); }
  struct Packed { u32 id; std::string data; };
  std::vector<Packed> packed;
  auto pack = [&](const std::vector<SaveCall::Col>& cols) { for (auto& c : cols) if (c.len > 0) packed.push_back({c.id, std::string((const char*)raw.data() + c.off, c.len)}); };
  pack(s.changeCols); const size_t numChangeCols = packed.size(); pack(s.opCols);
  if (!unknownCols.empty() && s.N > 0) {   // columns with ids this version does not know: host-encoded from the values kept per op (unknowncols.hpp)
    std::vector<std::pair<u32, std::string>> extra; appendUnknownDocColumns(extra);
    for (auto& e : extra) if (!e.second.empty()) packed.push_back({e.first, e.second});
    std::stable_sort(packed.begin() + numChangeCols, packed.end(), [](const Packed& a, const Packed& b) { return (a.id & ~8u) < (b.id & ~8u); });
  }
  {
    std::vector<std::thread> ts; std::vector<std::string> errs(packed.size());
    for (size_t k = 0; k < packed.size(); k++) if (packed[k].data.size() >= 256) ts.emplace_back([&, k] {
      try { packed[k].data = deflateRawBytes((const u8*)packed[k].data.data(), packed[k].data.size()); packed[k].id |= 8; } catch (Error& e) { errs[k] = e.what(); }
    });
    for (auto& t : ts) t.join();
    for (auto& e : errs) if (!e.empty()) throw Error(AMG_ERR_INTERNAL, e);   // the first in column order
  }
  trace.print("save", "columns deflated (host)", s.t0);
  std::string body;
  put_uleb(body, st.actorIds.size()); for (auto& a : st.actorIds) { put_uleb(body, a.size()); body += a; }
  put_uleb(body, st.heads.size()); for (auto& h : st.heads) body.append((const char*)h.data(), 32);
  put_uleb(body, numChangeCols); for (size_t k = 0; k < numChangeCols; k++) { put_uleb(body, packed[k].id); put_uleb(body, packed[k].data.size()); }
  put_uleb(body, packed.size() - numChangeCols); for (size_t k = numChangeCols; k < packed.size(); k++) { put_uleb(body, packed[k].id); put_uleb(body, packed[k].data.size()); }
  for (auto& p : packed) body += p.data;
  for (u32 i : st.headIdx) put_uleb(body, i);
  std::string hashed(1, '\0'); put_uleb(hashed, body.size()); hashed += body;
  u8 digest[32]; host_sha256((const u8*)hashed.data(), hashed.size(), digest);
  trace.print("save", "container assembled + hashed", s.t0);
  static const u8 magic[4] = {0x85, 0x6f, 0x4a, 0x83};
  result.assign((const char*)magic, 4); result.append((const char*)digest, 4); result += hashed;
}

// Backend.load(data) = new BackendDoc(buffer) (reference new.js:1709-1750): the document chunk's op columns are already in
// document order with succ lists, so loading = container check + column decode + one finalize pass. The container
// checksum (one SHA-256 over the whole chunk: inherently serial) and the DEFLATE of large columns are host pre-passes,
// as in SURVEY.md §2 row 12; column expansion and everything downstream run on the device.
inline void Engine::loadDocument(const u8* buf, size_t len) {
  if (numApplied != 0 || numRows != 0) throw Error(AMG_ERR_INTERNAL, "load needs a fresh backend");
  LoadCall l(buf, len);
  readContainer(l); inflateColumns(l); stageColumns(l); loadClock(l); countRows(l); decodeDocColumns(l); finalizeRows(l);
  readUnknownOpColumns(l); commitLoad(l);
  if (loaded.headIndexesUnknown) computeHashGraph();   // finds the heads' change indexes (and leaves the history rebuilt)
}

// container (columnar.js:688-708 decodeContainerHeader), document header and column directory (columnar.js:1006-1038 decodeDocumentHeader)
inline void Engine::readContainer(LoadCall& l) {
  const u8* buf = l.buf; const size_t len = l.len; ByteReader& r = l.r;
  if (len < 10 || buf[0] != 0x85 || buf[1] != 0x6f || buf[2] != 0x4a || buf[3] != 0x83) throw Error(AMG_ERR_RANGE, "Data does not begin with magic bytes 85 6f 4a 83");
  const u32 chunkType = buf[8]; r.pos = 9; const u64 chunkLen = r.uleb();
  if (r.err || (u64)r.pos + chunkLen > len) throw Error(AMG_ERR_RANGE, "buffer ended with incomplete number");
  u8 digest[32]; host_sha256(buf + 8, r.pos + (size_t)chunkLen - 8, digest);
  if (memcmp(digest, buf + 4, 4) != 0) throw Error(AMG_ERR_RANGE, "checksum does not match data");
  if ((u64)r.pos + chunkLen != len) throw Error(AMG_ERR_RANGE, "Encoded document has trailing data");
  if (chunkType != 0) throw Error(AMG_ERR_RANGE, "Unexpected chunk type: " + std::to_string(chunkType));
  trace.print("load", "container checksum", l.t0);
  const u64 numActors = r.uleb();
  for (u64 i = 0; i < numActors && !r.err; i++) { const u64 n = r.uleb(); if ((u64)r.pos + n > len) { r.err = KE_SUBARRAY; break; } l.actors.emplace_back((const char*)buf + r.pos, n); r.skip(n); }
  const u64 numHeads = r.uleb();
  for (u64 i = 0; i < numHeads && !r.err; i++) { if ((u64)r.pos + 32 > len) { r.err = KE_SUBARRAY; break; } std::array<u8, 32> h; memcpy(h.data(), buf + r.pos, 32); l.heads.push_back(h); r.skip(32); }
  auto readInfo = [&](std::vector<LoadCall::ColInfo>& cols) {
    const u64 n = r.uleb(); long long last = -1;
    for (u64 i = 0; i < n && !r.err; i++) { const u64 id = r.uleb(), cl = r.uleb(); if (last >= 0 && ((u32)id & ~8u) <= ((u32)last & ~8u)) throw Error(AMG_ERR_RANGE, "Columns must be in ascending order"); last = (long long)id; cols.push_back({(u32)id, cl, std::string()}); }
  };
  readInfo(l.changeCols); readInfo(l.opCols);
  auto readData = [&](std::vector<LoadCall::ColInfo>& cols) {
    for (auto& c : cols) {
      if (r.err || (u64)r.pos + c.len > len) throw Error(AMG_ERR_RANGE, "subarray exceeds buffer size");
      if (c.id & 8) l.deflated.emplace_back(&c, buf + r.pos); else c.data.assign((const char*)buf + r.pos, (size_t)c.len);
      r.skip(c.len);
    }
  };
  readData(l.changeCols); readData(l.opCols);
}

// DEFLATEd columns (columnar.js:1022-1027): independent streams, one host thread each when there are several large ones
inline void Engine::inflateColumns(LoadCall& l) {
  const auto& deflated = l.deflated;
  std::vector<std::string> errs(deflated.size()); std::vector<int> codes(deflated.size(), 0); std::vector<std::thread> ts;
  auto one = [&](size_t k) { try { LoadCall::ColInfo& c = *deflated[k].first; c.data = inflateRawBytes(deflated[k].second, (size_t)c.len); c.id ^= 8; } catch (Error& e) { errs[k] = e.what(); codes[k] = e.code; } catch (std::exception& e) { errs[k] = e.what(); codes[k] = AMG_ERR_INTERNAL; } };
  for (size_t k = 0; k < deflated.size(); k++) { if (deflated.size() > 1 && deflated[k].first->len >= (64u << 10)) ts.emplace_back(one, k); else one(k); }
  for (auto& t : ts) t.join();
  for (size_t k = 0; k < errs.size(); k++) if (codes[k]) throw Error(codes[k], errs[k]);   // the first in column order, as a sequential reader would meet it
  trace.print("load", "columns inflated", l.t0);
}

// actor ids, op columns and change metadata columns staged in the arena. First the head indexes that end the chunk: they
// are read only now so that an error of the inflate above wins over "buffer ended with incomplete number".
inline void Engine::stageColumns(LoadCall& l) {
  ByteReader& r = l.r;
  if (r.err) throw Error(AMG_ERR_RANGE, "buffer ended with incomplete number");
  if (!r.done()) for (size_t i = 0; i < l.heads.size(); i++) l.headIdx.push_back((u32)r.uleb());
  if (l.actors.size() > 65535) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 65535 actors in one document");
  hostArena.resize(0);
  { size_t total = 0; for (auto& a : l.actors) total += a.size(); for (auto& c : l.opCols) total += c.data.size(); for (auto& c : l.changeCols) total += c.data.size(); hostArena.reserve(total + 64); }   // one pinned allocation, not one per append
  for (auto& a : l.actors) { l.reps.emplace_back((u32)hostArena.size(), (u32)a.size()); hostArena.append(a.data(), a.size()); }
  for (auto& c : l.opCols) for (int k = 0; k < NUM_DOC_COLS; k++) if (c.id == DOC_COL_IDS[k]) { l.dc.off[k] = (u32)hostArena.size(); l.dc.len[k] = (u32)c.data.size(); hostArena.append(c.data.data(), c.data.size()); }
  // the change metadata columns stay available for a later save() (new.js:1717 keeps them as encoders)
  for (int k = 0; k < NUM_CHANGE_COLS; k++) l.doc.cols[k] = HostChange{(u32)hostArena.size(), 0};
  for (auto& c : l.changeCols) for (int k = 0; k < NUM_CHANGE_COLS; k++) if (c.id == CHANGE_COLS[k].id) { l.doc.cols[k] = HostChange{(u32)hostArena.size(), (u32)c.data.size()}; hostArena.append(c.data.data(), c.data.size()); }
  const size_t cur = l.arenaLen = hostArena.size();
  if (cur + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per document");
  arena.ensure(ctx, cur + 64); h2d(ctx, arena.p, hostArena.data(), cur); dev_memset(ctx, arena.p + cur, 0, 64);
  trace.print("load", "staged + uploaded", l.t0);
}

// change metadata: clock (new.js:1645-1675 readDocumentChanges). A long history is decoded and checked on the device
// (doccols.cuh + one stable sort by actor); a short one, or one the device path declines (malformed columns, a sequence
// error to report), by the same readers on the host, which produce the reference's error messages. Then the change index
// of every head.
inline void Engine::loadClock(LoadCall& l) {
  const std::vector<std::string>& actors = l.actors;
  l.clock.assign(actors.size(), 0); l.lastChange.assign(actors.size(), EMPTY32);
  bool onDevice = false; const HostChange ac = l.doc.cols[CC_ACTOR], sc = l.doc.cols[CC_SEQ]; u32 total = 0;
  if (ac.len >= parDocMinRows / 8 + 16 && sc.len > 0 && parCols.rleRecords(arena.p + ac.off, ac.len, &total) && total >= parDocMinRows) {
    const size_t n = total; DBuf<long long> aV, sV; aV.ensure(ctx, n + 1); sV.ensure(ctx, n + 1);
    if (parCols.toI64(arena.p + ac.off, ac.len, false, n, aV.p) && parCols.deltaToI64(arena.p + sc.off, sc.len, n, sV.p)) {
      sortKeys.ensure(ctx, n + 1); sortVals.ensure(ctx, n + 1); DBuf<u64> clkD; clkD.ensure(ctx, actors.size() + 1); dev_memset(ctx, clkD.p, 0, (actors.size() + 1) * 8);
      DBuf<u32> lastD; lastD.ensure(ctx, actors.size() + 1); dev_memset(ctx, lastD.p, 0xff, (actors.size() + 1) * 4);
      dev_memset(ctx, flagWord.p, 0, 16);
      foreach(ctx, n, ClockKeyKernel{aV.p, (u32)actors.size(), sortKeys.p, sortVals.p, flagWord.p});
      sortPairs(sortKeys, sortVals, n, bits_for(actors.size() > 1 ? actors.size() - 1 : 1));
      foreach(ctx, n, ClockCheckKernel{sortKeys.p, sortVals.p, sV.p, (u32)n, clkD.p, flagWord.p, lastD.p});
      u32 bad = 0; d2h(ctx, &bad, flagWord.p, 4); if (!actors.empty()) { d2h(ctx, l.clock.data(), clkD.p, actors.size() * 8); d2h(ctx, l.lastChange.data(), lastD.p, actors.size() * 4); } sync(ctx);
      if (!bad) { onDevice = true; l.doc.numChanges = n; } else { std::fill(l.clock.begin(), l.clock.end(), 0); std::fill(l.lastChange.begin(), l.lastChange.end(), EMPTY32); }
    }
  }
  if (!onDevice) {
    RleReader ar(hostArena.data() + ac.off, 0, ac.len, 0), sr(hostArena.data() + sc.off, 0, sc.len, 1); long long seqAcc = 0;   // (their staged copies)
    while (!ar.done()) {
      long long a = 0, d = 0; u32 o, n; const bool an = ar.next(a, o, n), sn = sr.next(d, o, n);
      if (ar.r.err || sr.r.err) throw Error(AMG_ERR_RANGE, "malformed change metadata columns");
      if (!an || (u64)a >= actors.size()) throw Error(AMG_ERR_RANGE, "actor index out of range");
      if (sn) seqAcc += d;
      const u64 seq = sn ? (u64)seqAcc : 0;
      if (seq != 1 && seq != l.clock[a] + 1) throw Error(AMG_ERR_RANGE, "Expected seq " + std::to_string(l.clock[a] + 1) + ", got " + std::to_string(seq) + " for actor " + hex_of((const u8*)actors[a].data(), actors[a].size()));
      l.clock[a] = seq; l.lastChange[a] = (u32)l.doc.numChanges++;
    }
  }
  trace.print("load", "clock", l.t0);
  if (!l.headIdx.empty() && l.headIdx.size() != l.heads.size()) l.headIdx.clear();
  // several heads without indexes (new.js:1734-1737: the hashes are known, their change indexes are not): the indexes are
  // found by reconstructing the change history right after the load (computeHashGraph)
  if (l.headIdx.empty()) { if (l.heads.size() == 1) l.headIdx.push_back((u32)(l.doc.numChanges ? l.doc.numChanges - 1 : 0)); else if (!l.heads.empty()) { l.doc.headIndexesUnknown = true; l.headIdx.assign(l.heads.size(), 0xffffffffu); } }
}

inline void Engine::ensureLoadRows(size_t n) {
  for (DBuf<u32>* b : {&r_objActor, &r_objCtr, &r_keyActor, &r_keyCtr, &r_keyStrOff, &r_keyStrLen, &r_insert, &r_action, &r_valLen, &r_valOff, &r_predNum, &r_predOff, &o_change, &o_time}) b->ensure(ctx, n + 1);
}

// Number of rows = values of the action column, number of succ entries = sum of succNum. Long columns take the parallel
// decoder (doccols.cuh); short, malformed or non-canonical ones the serial walkers, which also report the errors.
inline void Engine::countRows(LoadCall& l) {
  const DocCols& dc = l.dc;
  clearErr(); dev_memset(ctx, flagWord.p, 0, 16);
  { const char* e = getenv("AMG_PAR_DOC_MIN"); if (e) parDocMinRows = (size_t)strtoull(e, nullptr, 10); }
  auto succInParallel = [&](size_t rows) {   // many rows: the succ total in parallel too (succNum then needs no serial decode)
    if (rows < parDocMinRows || rows >= (1u << 29)) return;
    l.N = rows; ensureLoadRows(l.N); u64 sum = 0;
    if (dc.len[OC_SUCC_NUM] == 0) { l.counted = true; l.S = 0; }
    else if (parCols.countColumn(arena.p + dc.off[OC_SUCC_NUM], dc.len[OC_SUCC_NUM], l.N, r_predNum.p, r_predOff.p, &sum)) { l.counted = true; l.S = (size_t)sum; l.serialMask &= ~(1u << OC_SUCC_NUM); }
  };
  u32 total = 0;   // (a long column can still be a handful of records; then the serial count is instant anyway)
  if (dc.len[OC_ACTION] >= parDocMinRows / 8 + 16 && parCols.rleRecords(arena.p + dc.off[OC_ACTION], dc.len[OC_ACTION], &total)) succInParallel(total);
  if (!l.counted) {   // short action column: rows by the serial record walk
    foreach(ctx, 1, DocCountRowsKernel{arena.p, dc, flagWord.p, errWord.p});
    u32 n32 = 0; d2h(ctx, &n32, flagWord.p, 4); sync(ctx); checkErr();
    succInParallel(n32);
  }
  if (!l.counted) {
    foreach(ctx, 1, DocCountKernel{arena.p, dc, flagWord.p, errWord.p});
    u32 cnt[2]; d2h(ctx, cnt, flagWord.p, 8); sync(ctx); checkErr();
    l.N = cnt[0]; l.S = cnt[1];
  }
  trace.print("load", "rows counted", l.t0);
}

// Columns of a long document through the parallel decoders; what they decline, and every column of a short document,
// through DocColumnKernel (one launch, the columns selected by the mask).
inline void Engine::decodeDocColumns(LoadCall& l) {
  const size_t N = l.N, S = l.S; const DocCols& dc = l.dc;
  if (N >= (1u << 29)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^29 document rows");
  ensureLoadRows(N);
  r_predActor.ensure(ctx, S + 1); r_predCtr.ensure(ctx, S + 1);
  const RawRows raw = l.raw = rawRows();
  if (N >= parDocMinRows) {
    for (int k = 0; k < NUM_DOC_COLS; k++) {
      const int cx = doc_col_decoder(k);
      if (cx < 0 || !((l.serialMask >> k) & 1u)) continue;
      const size_t cnt = (cx == CX_PRED_ACTOR || cx == CX_PRED_CTR) ? S : N; const RawRows rr = doc_col_rows(k, raw, o_change.p, o_time.p); bool done = false;
      if (dc.len[k] == 0) {
        if (cnt > 0) foreach(ctx, cnt, DocAbsentKernel{cx, rr});
        done = true;
      } else if (cnt > 0) {   // (utf8 keys: below)
        u64 sum = 0;
        done = parCols.decode(CX_PAR_KIND[cx], arena.p + dc.off[k], dc.len[k], cnt, cx_outputs(rr, cx, 0, 0, dc.off[OC_VAL_RAW], &sum));
        if (cx == CX_VAL_LEN) done = done && sum <= dc.len[OC_VAL_RAW];
        if (cx == CX_PRED_NUM) done = done && sum == S;
      }
      if (done) l.serialMask &= ~(1u << k);
    }
    if ((l.serialMask >> OC_KEY_STR) & 1u) {   // keyStr: serial over records, parallel over rows
      DBuf<u32>& recStart = parCols.recOff; DBuf<u32>& recStrOff = parCols.recTok; DBuf<u32>& recStrLen = parCols.recN;
      recStart.ensure(ctx, N + 3); recStrOff.ensure(ctx, N + 3); recStrLen.ensure(ctx, N + 3);
      foreach_warp(ctx, 1, DocKeyStrRecordsKernel{arena.p, dc.off[OC_KEY_STR], dc.len[OC_KEY_STR], (u32)N, recStart.p, recStrOff.p, recStrLen.p, flagWord.p, errWord.p});
      u32 rc[2]; d2h(ctx, rc, flagWord.p, 8); sync(ctx); checkErr();
      foreach(ctx, N, DocKeyStrExpandKernel{recStart.p, recStrOff.p, recStrLen.p, rc[0], raw.keyStrOff, raw.keyStrLen});
      l.serialMask &= ~(1u << OC_KEY_STR);
    }
  }
  if (Trace::enabled()) fprintf(stderr, "amgpu load: %zu rows, %zu succ entries, columns left to the serial decoder: mask %04x (counted in parallel: %d)\n", N, S, l.serialMask & DECODED_DOC_COLS, l.counted ? 1 : 0);
  if (l.serialMask & DECODED_DOC_COLS) foreach_warp(ctx, NUM_DOC_COLS, DocColumnKernel{arena.p, dc, (u32)N, (u32)S, raw, o_change.p, o_time.p, errWord.p, l.serialMask});
  trace.print("load", "columns decoded", l.t0);
}

inline void Engine::finalizeRows(LoadCall& l) {
  const size_t N = l.N, S = l.S;
  doc.ensure(ctx, N + 1); succOff.ensure(ctx, N + 2); succ.ensure(ctx, S + 1);
  DBuf<u64>& maxOpD = pairSucc; maxOpD.ensure(ctx, 1); dev_memset(ctx, maxOpD.p, 0, 8);
  foreach(ctx, N, DocFinalizeKernel{l.raw, o_change.p, o_time.p, (u32)l.actors.size(), doc.view(), succOff.p, succ.p, maxOpD.p, errWord.p});
  { const u32 s32 = (u32)S; h2d(ctx, succOff.p + N, &s32, 4); }
  d2h(ctx, &l.maxOp, maxOpD.p, 8); sync(ctx); checkErr();
  trace.print("load", "rows finalized", l.t0);
}

// op columns with unknown ids: their values are kept per op (host; unknowncols.hpp) so that save() writes them again
inline void Engine::readUnknownOpColumns(LoadCall& l) {
  const size_t N = l.N;
  bool anyUnknown = false; for (auto& c : l.opCols) if (!is_known_doc_column(c.id)) anyUnknown = true;
  unknownCols.clear();
  if (!anyUnknown || N == 0) return;
  std::string all; std::vector<std::array<u32, 3>> cols;
  for (auto& c : l.opCols) { cols.push_back({c.id, (u32)all.size(), (u32)c.data.size()}); all += c.data; }
  std::vector<u64> ids(N); d2h(ctx, ids.data(), doc.id.p, N * 8); sync(ctx);
  const u32 e = read_unknown_columns((const u8*)all.data(), cols, N, is_known_doc_column, [&](size_t i, UnknownRow& row) {
    if (row.empty()) return;
    for (auto& kv : row) unknownCols.colIds.insert(kv.first);
    unknownCols.byOp[ids[i]] = row;
  });
  if (e == KE_UNSUPPORTED_OP) throw Error(AMG_ERR_RANGE, "unexpected VALUE_RAW column");
  if (e) throwKernelError((u64)e);
}

// change history placeholders: only the head hashes are known (new.js:1727-1739); then the document's host state
inline void Engine::commitLoad(LoadCall& l) {
  const size_t numChanges = l.doc.numChanges; const auto& hs = l.heads;
  hashes.ensure(ctx, numChanges * 32 + 64); dev_memset(ctx, hashes.p, 0, numChanges * 32 + 64);
  if (!l.doc.headIndexesUnknown) for (size_t i = 0; i < hs.size(); i++) { if (l.headIdx[i] >= numChanges) throw Error(AMG_ERR_RANGE, "head index out of range"); h2d(ctx, hashes.p + (size_t)l.headIdx[i] * 32, hs[i].data(), 32); }
  sync(ctx);
  numRows = l.N; numSucc = l.S; numApplied = numChanges; arenaLen = l.arenaLen;
  std::vector<size_t> o(hs.size()); for (size_t i = 0; i < o.size(); i++) o[i] = i; std::sort(o.begin(), o.end(), [&](size_t a, size_t b) { return hs[a] < hs[b]; });
  st = DocState{l.actors, l.reps, l.clock, l.maxOp, {}, {}}; for (size_t i : o) { st.heads.push_back(hs[i]); st.headIdx.push_back(l.headIdx[i]); }
  changes.assign(numChanges, HostChange{0, 0});
  lastChange.ensure(ctx, st.actorIds.size() + 1); h2d(ctx, lastChange.p, l.lastChange.data(), st.actorIds.size() * 4);
  l.doc.bytes.assign((const char*)l.buf, l.len); l.doc.haveHashGraph = false; loaded = std::move(l.doc);
  trace.print("load", "host state", l.t0);
  while (actorCap < 2 * (st.actorIds.size() + 16)) actorCap *= 2;
  actorSlots.ensure(ctx, actorCap); rebuildActorTable();
}

// ---------------------------------------------------------------- device spans (amg_last_*_ms)
inline void DeviceSpans::resume(SpanKind k) {
  kind = k;
#ifndef AMG_EMU
  if (!ev[0]) for (auto& e : ev) CUDA_CHECK(cudaEventCreate(&e));
  CUDA_CHECK(cudaEventRecord(ev[0], ctx.stream));
#endif
}
inline void DeviceSpans::stop() {
#ifndef AMG_EMU
  float t = 0; CUDA_CHECK(cudaEventRecord(ev[1], ctx.stream));
  CUDA_CHECK(cudaEventSynchronize(ev[1])); CUDA_CHECK(cudaEventElapsedTime(&t, ev[0], ev[1])); ms[kind] += t;
#endif
}

// ---------------------------------------------------------------- sync protocol (sync.js:234-306)
inline void Engine::uploadCandidates(const u32* idx, size_t count) {
  if (!idx) return;
  syncIdx.ensure(ctx, count + 1); h2d(ctx, syncIdx.p, idx, count * 4);
}

// makeBloomFilter (sync.js:234-238): BloomFilter(hashes).bytes = LEB128 numEntries, 10, 7, then ceil(10 * count / 8) bytes
inline void Engine::syncBloom(const u32* idx, size_t count, std::string& out) {
  out.clear(); spans.start(SPAN_SYNC);
  if (count == 0) return;   // BloomFilter([]).bytes is empty
  const size_t bitsBytes = (BLOOM_BITS_PER_ENTRY * count + 7) / 8, words = (bitsBytes + 3) / 4;
  uploadCandidates(idx, count);
  syncBits.ensure(ctx, words); dev_memset(ctx, syncBits.p, 0, words * 4);
  foreach(ctx, count, BloomAddKernel{hashes.p, idx ? syncIdx.p : nullptr, 8 * (u64)bitsBytes, syncBits.p});
  put_uleb(out, count); put_uleb(out, BLOOM_BITS_PER_ENTRY); put_uleb(out, BLOOM_NUM_PROBES);
  const size_t at = out.size(); out.resize(at + words * 4);
  d2h(ctx, &out[at], syncBits.p, words * 4); sync(ctx);
  out.resize(at + bitsBytes);
  spans.stop();
}

// getChangesToSend (sync.js:246-306) for a non-empty `have`: which candidates go out because of the peer's filters.
inline void Engine::syncChangesToSend(const u32* idx, size_t count, const std::vector<BloomSpec>& filters, std::vector<u8>& send) {
  send.assign(count, 0); spans.start(SPAN_SYNC);
  if (count == 0) return;
  for (auto& f : filters)
    if (f.numProbes > BLOOM_MAX_PROBES) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: a Bloom filter with " + std::to_string(f.numProbes) + " probes (the device path takes at most " + std::to_string(BLOOM_MAX_PROBES) + ")");
  uploadCandidates(idx, count);
  const u32* idxD = idx ? syncIdx.p : nullptr;
  // sync.js:273-276: a candidate is negative when no filter contains it
  std::vector<BloomRef> refs; std::string blob;
  for (auto& f : filters) {
    const bool empty = f.numEntries == 0 || f.bitsLen == 0;
    refs.push_back(BloomRef{blob.size(), empty ? 0 : 8 * (u64)f.bitsLen, f.numProbes, 0});
    if (!empty) blob.append((const char*)f.bits, f.bitsLen);
  }
  syncFilters.ensure(ctx, refs.size() + 1); h2d(ctx, syncFilters.p, refs.data(), refs.size() * sizeof(BloomRef));
  syncFilterBits.ensure(ctx, blob.size() + 1); h2d(ctx, syncFilterBits.p, blob.data(), blob.size());
  syncNeg.ensure(ctx, count);
  foreach(ctx, count, BloomProbeKernel{hashes.p, idxD, syncFilterBits.p, syncFilters.p, (u32)refs.size(), syncNeg.p});
  d2h(ctx, send.data(), syncNeg.p, count); sync(ctx);
  size_t numNeg = 0; for (u8 v : send) numNeg += v;
  if (numNeg == 0 || numNeg == count) { spans.stop(); return; }   // a peer that has everything, or a new one: no closure needed
  // sync.js:277-289: everything that depends on a Bloom-negative candidate goes too. The candidates' dependency indexes are
  // resolved like save() does (parseChangeHeaders, resolveChangeDeps).
  const size_t K = count, C = numApplied;
  std::vector<HostChange> pairs(K); for (size_t i = 0; i < K; i++) pairs[i] = changes[idx ? idx[i] : i];
  clearErr();
  const u32 totalDeps = parseChangeHeaders(arena.p, pairs.data(), K);
  checkErr();
  resolveChangeDeps(arena.p, hashes.p, C, K, 0, totalDeps);
  std::vector<u32> base(K + 1), deps(totalDeps);
  d2h(ctx, base.data(), depBase.p, (K + 1) * 4); d2h(ctx, deps.data(), depIdx.p, (size_t)totalDeps * 4); sync(ctx);
  spans.stop();
  // One forward pass in application order: a change is applied only after its dependencies (a loaded document stores its
  // changes in topological order), so a candidate's candidate dependencies are decided before it is. This stays on the host
  // on purpose: it is O(candidates + deps), while a device frontier walk needs one launch per dependency level, which on a
  // history that is one long chain is one launch per change (up to 10^6).
  std::vector<u32> order(K); for (size_t i = 0; i < K; i++) order[i] = (u32)i;
  if (idx) std::sort(order.begin(), order.end(), [&](u32 a, u32 b) { return idx[a] < idx[b]; });
  std::vector<u8> marked(C, 0);   // by change index; only candidates are ever marked
  for (u32 p : order) {
    u8 m = send[p];
    for (u32 j = base[p]; j < base[p + 1] && !m; j++) if (deps[j] != DEP_MISSING && marked[deps[j]]) m = 1;
    send[p] = m; marked[idx ? idx[p] : p] = m;
  }
}

// ------------------------------------------------------------ decodeChange / decodeChanges (changes.cuh)
inline void Engine::decodeChanges(const u8* blob, const u64* offsets, size_t n, bool history, std::string& out) {
  DecodeCall d; d.n = n; d.history = history; decodeFailed = 0;
  spans.start(SPAN_DECODE);
  dcErr.ensure(ctx, DP_NUM); dev_memset(ctx, dcErr.p, 0, DP_NUM * 8);
  clearErr();
  dcOff.ensure(ctx, n + 1); dcLen.ensure(ctx, n + 1); dcHash.ensure(ctx, n * 32 + 64);
  if (history) {   // every applied change (getAllChanges order), inflated copies in place; their hashes are the engine's
    computeHashGraph();
    if (n) {
      chPairs.ensure(ctx, n); h2d(ctx, chPairs.p, changes.data(), n * sizeof(HostChange));
      foreach(ctx, n, SplitPairsKernel{chPairs.p, dcOff.p, dcLen.p});
      d2d(ctx, dcHash.p, hashes.p, n * 32);
    }
    d.ar = arena.p;
  } else {
    stageDecodeInput(d, blob, offsets);
    inflateDecodeInput(d);
    d.ar = dcArena.p;
  }
  decodeTable(d, out);
  spans.stop();
}

// the caller's bytes into scratch (never into the document's arena): device memory is copied device to device, host
// memory (pinned or pageable) uploaded
inline void Engine::stageDecodeInput(DecodeCall& d, const u8* blob, const u64* offsets) {
  const size_t n = d.n; const u64 total = n ? offsets[n] - offsets[0] : 0;
  if (total + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per call");
  dcArena.ensure(ctx, total + 64);
  bool onDevice = false;
#ifndef AMG_EMU
  if (n) { cudaPointerAttributes at; if (cudaPointerGetAttributes(&at, blob + offsets[0]) == cudaSuccess) onDevice = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged; else cudaGetLastError(); }
#endif
  if (onDevice) d2d(ctx, dcArena.p, blob + offsets[0], total); else h2d(ctx, dcArena.p, blob + offsets[0], total);
  dev_memset(ctx, dcArena.p + total, 0, 64);
  std::vector<u32> ol(2 * n + 2);
  for (size_t i = 0; i < n; i++) { ol[i] = (u32)(offsets[i] - offsets[0]); ol[n + i] = (u32)(offsets[i + 1] - offsets[i]); }
  h2d(ctx, dcOff.p, ol.data(), n * 4); h2d(ctx, dcLen.p, ol.data() + n, n * 4);
  d.tot[3] = (u32)total;   // bytes staged so far: DEFLATEd changes are inflated behind them
}

// DEFLATEd entries (columnar.js:742) inflated on the device, behind the staged bytes: the sequence of inflateBatch (flag ->
// scan -> list -> k_inflate into scratch -> scan -> k_inflate in place). Their offsets are re-pointed to the inflated copies.
inline void Engine::inflateDecodeInput(DecodeCall& d) {
  const size_t B = d.n; if (B == 0) return;
  emit.ensure(ctx, B + 1); slot.ensure(ctx, B + 2); dcDefl.ensure(ctx, B + 1);   // (own list: benchDecode re-reads the apply path's deflList)
  dev_memset(ctx, flagWord.p + 8, 0, 4);
  foreach(ctx, B, DeflateFlagKernel{dcArena.p, dcOff.p, dcLen.p, emit.p, flagWord.p + 8});
  scan_exclusive(ctx, scanTmp, emit.p, slot.p, B);
  u32 nd32 = 0, deflBytes = 0; readU32x2(slot.p + B, flagWord.p + 8, &nd32, &deflBytes);
  const size_t nd = nd32; if (nd == 0) return;
  foreach(ctx, B, CompactKernel{emit.p, slot.p, dcDefl.p});
  inflLen.ensure(ctx, nd + 1); inflOff.ensure(ctx, nd + 2); patchTriples.ensure(ctx, 2 * nd + 2); inflCap.ensure(ctx, nd + 2); inflCapOff.ensure(ctx, nd + 2); inflOvf.ensure(ctx, nd + 1);
  u32 factor = 4; while (factor > 1 && (u64)factor * deflBytes + 1024ull * nd >= 0xf0000000ULL) factor--;
  inflScratch.ensure(ctx, (size_t)factor * deflBytes + 1024 * nd + 64);
  foreach(ctx, nd, InflateCapKernel{dcDefl.p, dcLen.p, factor, inflCap.p});
  scan_exclusive(ctx, scanTmp, inflCap.p, inflCapOff.p, nd);
  InflateArgs ia{dcArena.p, dcOff.p, dcLen.p, dcDefl.p, nd, inflLen.p, nullptr, 0u, patchTriples.p, patchTriples.p + nd, inflScratch.p, inflCapOff.p, inflOvf.p, dcErr.p + DP_INFLATE};
  const u64 extra = inflateSpeculate(ia); const size_t start = d.tot[3];
  if ((u64)start + extra + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per call");
  dcArena.ensure(ctx, start + extra + 64, start);
  ia.arena = dcArena.p; ia.outOff = inflOff.p; ia.extraStart = (u32)start;
  inflate_changes(ctx, INFL_PLACE, ia);
  dev_memset(ctx, dcArena.p + start + extra, 0, 64);
  foreach(ctx, nd, InflatePatchKernel{dcDefl.p, inflLen.p, inflOff.p, (u32)start, dcOff.p, dcLen.p});
  d.tot[3] = (u32)(start + extra);
}

inline void Engine::decodeTable(DecodeCall& d, std::string& out) {
  const size_t n = d.n; const u8* ar = d.ar;
  dcCLen.ensure(ctx, n + 1); dcMeta.ensure(ctx, n + 1); dcColOff.ensure(ctx, (size_t)CHG_COLS * n + 1); dcColLen.ensure(ctx, (size_t)CHG_COLS * n + 1);
  for (auto* b : {&dcOps, &dcPreds, &dcActors, &dcBytes, &dcOpBase, &dcPredBase, &dcActorBase, &dcByteBase}) b->ensure(ctx, n + 2);
  foreach(ctx, n, ChgContainerKernel{ar, dcOff.p, dcLen.p, dcCLen.p, dcErr.p + DP_CONTAINER});
  if (!d.history) foreach(ctx, n, ShaKernel{ar, dcOff.p, dcCLen.p, dcHash.p, dcErr.p + DP_SHA, nullptr, nullptr});
  foreach(ctx, n, ChgHeaderKernel{ar, dcOff.p, dcLen.p, dcCLen.p, dcHash.p, dcMeta.p, dcColOff.p, dcColLen.p, dcOps.p, dcPreds.p, dcActors.p, dcBytes.p, n, dcErr.p + DP_HEADER});
  scan_exclusive(ctx, scanTmp, dcOps.p, dcOpBase.p, n); scan_exclusive(ctx, scanTmp, dcPreds.p, dcPredBase.p, n);
  scan_exclusive(ctx, scanTmp, dcActors.p, dcActorBase.p, n); scan_exclusive(ctx, scanTmp, dcBytes.p, dcByteBase.p, n);
  // the scans are 32-bit: their totals are only used once the 64-bit sums show that nothing wrapped (bytes: at most the
  // staged input or the arena, both below 4 GiB)
  dcTotals.ensure(ctx, 3); dev_memset(ctx, dcTotals.p, 0, 3 * 8);
  foreach(ctx, n, ChgTotalsKernel{dcOps.p, dcPreds.p, dcActors.p, dcTotals.p});
  u64 t64[3] = {0, 0, 0}; void* dst[4] = {&t64[0], &t64[1], &t64[2], &d.tot[3]};
  readWords({{dcTotals.p, 8}, {dcTotals.p + 1, 8}, {dcTotals.p + 2, 8}, {dcByteBase.p + n, 4}}, dst);
  if (t64[0] >= 0x7fffffffULL || t64[1] >= 0x7fffffffULL || t64[2] >= 0x7fffffffULL)
    throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^31 operations, preds or actor table entries in one decodeChanges call");
  for (int k = 0; k < 3; k++) d.tot[k] = (u32)t64[k];
  const size_t M = d.tot[0], P = d.tot[1], A = d.tot[2], Bt = d.tot[3];
  auto align8 = [](size_t v) { return (v + 7) & ~(size_t)7; };
  d.changesOff = CHG_HDR_WORDS * 8; d.opsOff = d.changesOff + n * sizeof(ChangeRec); d.predsOff = d.opsOff + M * sizeof(OpRec);
  d.actorsOff = d.predsOff + P * 8; d.bytesOff = d.actorsOff + A * sizeof(ActorRef); d.size = align8(d.bytesOff + Bt);
  if (d.size >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: a change table is limited to 4 GiB");
  dcOut.ensure(ctx, d.size + 64);
  const u64 hdr[CHG_HDR_WORDS] = {CHG_MAGIC, n, d.changesOff, M, d.opsOff, P, d.predsOff, A, d.actorsOff, d.bytesOff, Bt, 0};
  h2d(ctx, dcOut.p, hdr, sizeof(hdr)); sync(ctx);   // (hdr lives on this stack frame)
  // SoA rows: the 12 columns of RawRows over M ops, then predActor / predCtr over P preds; child columns
  dcRows.ensure(ctx, 12 * (M + 1) + 2 * (P + 1)); dcChld.ensure(ctx, 2 * (M + 1));
  u32* r = dcRows.p; const size_t Ms = M + 1;
  RawRows raw{r, r + Ms, r + 2 * Ms, r + 3 * Ms, r + 4 * Ms, r + 5 * Ms, r + 6 * Ms, r + 7 * Ms, r + 8 * Ms, r + 9 * Ms, r + 10 * Ms, r + 11 * Ms, r + 12 * Ms, r + 12 * Ms + P + 1};
  foreach(ctx, (size_t)NCOLS * n, ChgColumnsKernel{ar, dcColOff.p, dcColLen.p, dcOps.p, dcPreds.p, dcOpBase.p, dcPredBase.p, n, raw, dcChld.p, dcChld.p + Ms, dcErr.p + DP_COLUMNS});
  u8* o = dcOut.p;
  foreach(ctx, n, ChgRecordKernel{ar, dcMeta.p, dcHash.p, dcOps.p, dcActors.p, dcOpBase.p, dcPredBase.p, dcActorBase.p, dcByteBase.p, (u64)d.bytesOff,
                                  reinterpret_cast<ChangeRec*>(o + d.changesOff), reinterpret_cast<ActorRef*>(o + d.actorsOff)});
  foreach(ctx, (Bt + 63) / 64, ChgBytesKernel{ar, dcOff.p, dcByteBase.p, n, (u32)Bt, o + d.bytesOff});
  foreach(ctx, M, ChgOpKernel{ar, dcOff.p, dcOpBase.p, n, raw, dcChld.p, dcChld.p + Ms, dcColOff.p, dcColLen.p, dcActors.p, dcActorBase.p, dcByteBase.p, (u64)d.bytesOff,
                              o, reinterpret_cast<const ActorRef*>(o + d.actorsOff), reinterpret_cast<OpRec*>(o + d.opsOff), reinterpret_cast<u32*>(o + d.predsOff), dcErr.p + DP_OPS});
  u64 w[DP_NUM] = {0}; void* wd[DP_NUM]; for (int k = 0; k < DP_NUM; k++) wd[k] = &w[k];
  readWords({{dcErr.p, 8}, {dcErr.p + 1, 8}, {dcErr.p + 2, 8}, {dcErr.p + 3, 8}, {dcErr.p + 4, 8}, {dcErr.p + 5, 8}}, wd);
  for (int k = 0; k < DP_NUM; k++) if (w[k]) throwDecodeError(d, w);
  out.resize(d.size);
  d2h(ctx, &out[0], dcOut.p, d.size); sync(ctx);
}

// The change the sequential reference fails on first: the smallest failing change over the phases' error words (those of
// phase opPhase are keyed by op and mapped to their change through the n + 1 op offsets at opBaseDev), and its earliest
// failing phase
inline std::pair<size_t, int> Engine::firstFailingChange(const u64* w, int numPhases, int opPhase, const u32* opBaseDev, size_t n) {
  std::vector<u32> opBase(n + 1); d2h(ctx, opBase.data(), opBaseDev, (n + 1) * 4); sync(ctx);
  size_t best = SIZE_MAX; int phase = -1;
  for (int k = 0; k < numPhases; k++) {
    if (!w[k]) continue;
    size_t c = (size_t)(w[k] >> 8);
    if (k == opPhase) c = (size_t)(std::upper_bound(opBase.begin(), opBase.end(), (u32)c) - opBase.begin()) - 1;
    if (c < best) { best = c; phase = k; }
  }
  return {best, phase};
}

// The first failing change (firstFailingChange), and for it the error of its earliest phase
inline void Engine::throwDecodeError(DecodeCall& d, const u64* w) {
  const auto [best, phase] = firstFailingChange(w, DP_NUM, DP_OPS, dcOpBase.p, d.n);
  decodeFailed = best; const u32 code = (u32)(w[phase] & 0xff);
  auto actorIndex = [](u32 a) { return "No actor index " + std::to_string(a); };
  if (code == DE_CHUNK_TYPE_N) {
    u32 off = 0; d2h(ctx, &off, dcOff.p + best, 4); sync(ctx); u8 t = 0; d2h(ctx, &t, d.ar + off + 8, 1); sync(ctx);
    throw Error(AMG_ERR_RANGE, "Unexpected chunk type: " + std::to_string(t));
  }
  if (phase == DP_OPS) {
    const size_t g = (size_t)(w[phase] >> 8); OpRec o; d2h(ctx, &o, dcOut.p + d.opsOff + g * sizeof(OpRec), sizeof(OpRec)); sync(ctx);
    auto txt = [](u32 v) { return v == NULL32 ? std::string("None") : std::to_string(v); };
    switch (code) {
      case DE_OBJ_ACTOR: throw Error(AMG_ERR_RANGE, actorIndex(o.objActor));
      case DE_KEY_ACTOR: throw Error(AMG_ERR_RANGE, actorIndex(o.keyActor));
      case DE_CHLD_ACTOR: throw Error(AMG_ERR_RANGE, actorIndex(o.chldActor));
      case DE_PRED_ACTOR: {
        std::vector<u32> pr(2 * (size_t)o.predNum + 2); d2h(ctx, pr.data(), dcOut.p + d.predsOff + (size_t)o.predFirst * 8, (size_t)o.predNum * 8);
        u32 na = 0; d2h(ctx, &na, dcActors.p + o.change, 4); sync(ctx);
        for (u32 j = 0; j < o.predNum; j++) if (pr[2 * j] != NULL32 && pr[2 * j] >= na) throw Error(AMG_ERR_RANGE, actorIndex(pr[2 * j]));
        break;
      }
      case DE_CHLD_MISMATCH: throw Error(AMG_ERR_RANGE, "Mismatched child columns: " + txt(o.chldCtr) + " and " + txt(o.chldActor));
      case DE_PRED_ORDER: throw Error(AMG_ERR_RANGE, "operation IDs are not in ascending order");
      case DE_PRED_NULL: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: a pred list that orders a null operation ID (the reference compares null with a number)");
      case KE_FLOAT_LEN: throw Error(AMG_ERR_RANGE, "Invalid length for floating point number: " + std::to_string(o.valLen >> 4));
      default: break;
    }
  }
  throwKernelError(w[phase]);
}

// ------------------------------------------------------------ encodeChange over a change table (encchg.cuh)
inline void Engine::encodeChanges(const u8* table, size_t len, std::string& out, std::vector<u64>& offs, std::string& hashesOut) {
  EncodeCall e; e.len = len; encodeFailed = 0;
  spans.start(SPAN_ENCODE);
  clearErr();
  stageEncodeInput(e, table);
  if (e.n) { validateTable(e); encodeActorTables(e); encodePrep(e); encodeColumns(e); encodeHashes(e); }
  copyEncodeOutput(e, out, offs, hashesOut);
  spans.stop();
}

// 1. the table into scratch as decodeChanges stages its input (pinned, pageable or device memory); the header's sections
// checked on the host: inside the table and aligned for their records
inline void Engine::stageEncodeInput(EncodeCall& e, const u8* table) {
  auto bad = [](const std::string& what) { throw Error(AMG_ERR_RANGE, "change table: " + what); };
  if (e.len < CHG_HDR_WORDS * 8) bad("shorter than its header");
  DecodeCall d; d.n = 1; const u64 offs[2] = {0, (u64)e.len};
  dcOff.ensure(ctx, 2); dcLen.ensure(ctx, 2);
  stageDecodeInput(d, table, offs);
  d2h(ctx, e.hdr, dcArena.p, sizeof(e.hdr)); sync(ctx);
  const u64* h = e.hdr;
  if (h[0] != CHG_MAGIC) bad("bad magic");
  auto section = [&](u64 count, u64 off, u64 size, u64 align, const char* what) {
    if (off % align || off > e.len || count > (e.len - off) / size) bad(std::string(what) + " section out of range");
  };
  section(h[1], h[2], sizeof(ChangeRec), 8, "changes"); section(h[3], h[4], sizeof(OpRec), 8, "ops");
  section(h[5], h[6], 8, 4, "preds"); section(h[7], h[8], sizeof(ActorRef), 4, "actors");
  e.n = (size_t)h[1];
  const u8* t = dcArena.p;
  e.T = EncTable{t, e.len, h[3], h[5], h[7], reinterpret_cast<const ChangeRec*>(t + h[2]), reinterpret_cast<const OpRec*>(t + h[4]),
                 reinterpret_cast<const u32*>(t + h[6]), reinterpret_cast<const ActorRef*>(t + h[8])};
}

// 2. change records (thread per change), then ops (thread per op); every error of the call is known before anything is sized
inline void Engine::validateTable(EncodeCall& e) {
  const size_t n = e.n;
  e.err.ensure(ctx, EP_NUM); dev_memset(ctx, e.err.p, 0, EP_NUM * 8);
  e.totals.ensure(ctx, 4); dev_memset(ctx, e.totals.p, 0, 4 * 8);
  for (auto* b : {&e.nOps, &e.nPreds, &e.nActors, &e.opBase, &e.predBase, &e.actorBase}) b->ensure(ctx, n + 2);
  foreach(ctx, n, EncChangeKernel{e.T, e.nOps.p, e.nPreds.p, e.nActors.p, reinterpret_cast<u32*>(e.totals.p + 3), e.err.p + EP_CHANGES, e.err.p + EP_SIZE});
  foreach(ctx, n, ChgTotalsKernel{e.nOps.p, e.nPreds.p, e.nActors.p, e.totals.p});
  u64 t[4] = {0, 0, 0, 0}; void* dst[4] = {&t[0], &t[1], &t[2], &t[3]};
  readWords({{e.totals.p, 8}, {e.totals.p + 1, 8}, {e.totals.p + 2, 8}, {e.totals.p + 3, 8}}, dst);
  // the scans are 32-bit, and every op takes 3 + predNum actor slots
  if (t[0] >= 0x7fffffffULL || t[1] >= 0x7fffffffULL || t[2] >= 0x7fffffffULL || 3 * t[0] + t[1] >= 0x7fffffffULL)
    throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^31 operations, preds or actor table entries in one encodeChanges call");
  e.M = t[0]; e.P = t[1]; e.E = t[2]; e.maxActorLen = (u32)t[3];
  scan_exclusive(ctx, scanTmp, e.nOps.p, e.opBase.p, n); scan_exclusive(ctx, scanTmp, e.nPreds.p, e.predBase.p, n); scan_exclusive(ctx, scanTmp, e.nActors.p, e.actorBase.p, n);
  e.slotCnt.ensure(ctx, e.M + 2); e.slotBase.ensure(ctx, e.M + 3);
  if (e.M) foreach(ctx, e.M, EncOpKernel{e.T, e.opBase.p, n, e.slotCnt.p, e.err.p + EP_OPS});
  u64 w[EP_NUM] = {0, 0, 0}; void* wd[EP_NUM] = {&w[0], &w[1], &w[2]};
  readWords({{e.err.p, 8}, {e.err.p + 1, 8}, {e.err.p + 2, 8}}, wd);
  if (w[EP_CHANGES] || w[EP_OPS] || w[EP_SIZE]) throwEncodeError(e, w);   // nothing is sized before every change is known to fit
}

// 3. actor ids ranked over the call (LSD radix sort: length, then 8-byte chunks from the last), then every change's other
// actors: its sorted, unique (change, rank) pairs (the history kernels)
inline void Engine::encodeActorTables(EncodeCall& e) {
  const size_t n = e.n, E = e.E, M = e.M;   // (every change has its author: E >= n > 0)
  for (auto* b : {&e.entOff, &e.entLen, &e.entRank, &e.rep, &e.head, &e.headScan}) b->ensure(ctx, E + 2);
  e.sortKeys.ensure(ctx, E + 1); e.sortVals.ensure(ctx, E + 1);
  foreach(ctx, n, EncActorListKernel{e.T, e.nActors.p, e.actorBase.p, e.entOff.p, e.entLen.p});
  foreach(ctx, E, EncActorKeyKernel{e.T.t, e.entOff.p, e.entLen.p, nullptr, -1, e.sortKeys.p, e.sortVals.p});
  radix_sort_pairs(ctx, sortTmp, e.sortKeys, e.sortVals, E, 0, bits_for(e.maxActorLen));
  for (int q = (int)((e.maxActorLen + 7) / 8) - 1; q >= 0; q--) {
    foreach(ctx, E, EncActorKeyKernel{e.T.t, e.entOff.p, e.entLen.p, e.sortVals.p, q, e.sortKeys.p, nullptr});
    radix_sort_pairs(ctx, sortTmp, e.sortKeys, e.sortVals, E, 0, 64);
  }
  foreach(ctx, E, EncActorHeadKernel{e.T.t, e.entOff.p, e.entLen.p, e.sortVals.p, e.head.p});
  scan_exclusive(ctx, scanTmp, e.head.p, e.headScan.p, E);
  foreach(ctx, E, EncActorRankKernel{e.sortVals.p, e.head.p, e.headScan.p, e.entRank.p, e.rep.p});
  if (M) { scan_exclusive(ctx, scanTmp, e.slotCnt.p, e.slotBase.p, M); e.Q = readU32(e.slotBase.p + M); }
  const size_t Q = e.Q;
  e.slotKeys.ensure(ctx, Q + 1); e.sortVals.ensure(ctx, Q + 1); e.uniq.ensure(ctx, Q + 2); e.uniqSlot.ensure(ctx, Q + 3);
  if (Q) {
    foreach(ctx, M, EncActorPairKernel{e.T, e.opBase.p, n, e.actorBase.p, e.entRank.p, e.slotBase.p, e.slotKeys.p});
    foreach(ctx, Q, HistIotaKernel{e.sortVals.p});
    radix_sort_pairs(ctx, sortTmp, e.slotKeys, e.sortVals, Q, 0, std::min(64, 32 + bits_for(n)));   // (~0 = no actor: all ones, sorts last)
    foreach(ctx, Q, HistUniqueKernel{e.slotKeys.p, e.uniq.p});
    scan_exclusive(ctx, scanTmp, e.uniq.p, e.uniqSlot.p, Q);
    e.U = readU32(e.uniqSlot.p + Q);
  }
  e.other.ensure(ctx, e.U + 1); e.otherStart.ensure(ctx, n + 2);
  if (e.U) foreach(ctx, Q, HistOtherFillKernel{e.slotKeys.p, e.uniq.p, e.uniqSlot.p, e.other.p});
  foreach(ctx, n + 1, HistLowerBoundKernel{e.other.p, (u32)e.U, 32, e.otherStart.p});
}

// 4. local actor numbers, delta values, sorted preds (thread per change)
inline void Engine::encodePrep(EncodeCall& e) {
  const size_t M = e.M, P = e.P;
  for (auto* b : {&e.objA, &e.keyA, &e.chA}) b->ensure(ctx, M + 1);
  for (auto* b : {&e.keyDelta, &e.chDelta}) b->ensure(ctx, M + 1);
  e.predA.ensure(ctx, P + 1); e.predDelta.ensure(ctx, P + 1); e.predKey.ensure(ctx, P + 1);
  foreach(ctx, e.n, EncPrepKernel{e.T, e.opBase.p, e.predBase.p, e.actorBase.p, e.entRank.p, e.other.p, e.otherStart.p, e.objA.p, e.keyA.p, e.keyDelta.p, e.chA.p, e.chDelta.p,
                                  e.predKey.p, e.predA.p, e.predDelta.p});
}

// 5. column lengths (thread per (column, change)), container lengths, offsets (64-bit scan), headers, then the columns
inline void Engine::encodeColumns(EncodeCall& e) {
  const size_t n = e.n;
  const EncCols cols{e.opBase.p, e.predBase.p, e.objA.p, e.keyA.p, e.keyDelta.p, e.chA.p, e.chDelta.p, e.predA.p, e.predDelta.p};
  e.colLen.ensure(ctx, (size_t)HC_NUM * n + 1); e.outLen.ensure(ctx, n + 1); e.outOff.ensure(ctx, n + 2);
  for (auto* b : {&e.dataAt, &e.depsAt, &e.bodyAt}) b->ensure(ctx, n + 1);
  foreach(ctx, (size_t)HC_NUM * n, EncColSizeKernel{e.T, cols, n, e.colLen.p});
  EncChangeHeadKernel hk{0, e.T, n, e.colLen.p, e.actorBase.p, e.entOff.p, e.entLen.p, e.rep.p, e.other.p, e.otherStart.p, e.outLen.p, e.outOff.p, nullptr, e.dataAt.p, e.depsAt.p, e.bodyAt.p};
  foreach(ctx, n, hk);
  scan_exclusive64(ctx, scanTmp, EncOutLen64{e.outLen.p}, e.outOff.p, n);
  u64 total = 0; void* dst[1] = {&total}; readWords({{e.outOff.p + n, 8}}, dst);
  if (total + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: the changes of one encodeChanges call are limited to 4 GiB");
  e.total = total; e.out.ensure(ctx, total + 64);
  hk.pass = 1; hk.out = e.out.p; foreach(ctx, n, hk);
  foreach(ctx, (size_t)HC_NUM * n, EncColWriteKernel{e.T, cols, n, e.colLen.p, e.dataAt.p, e.out.p});
}

// 6. hashes and checksums (thread per change: the dependencies are given as hashes)
inline void Engine::encodeHashes(EncodeCall& e) {
  e.hashes.ensure(ctx, e.n * 32 + 64);
  foreach(ctx, e.n, EncHashKernel{e.T, e.outOff.p, e.outLen.p, e.depsAt.p, e.bodyAt.p, e.out.p, e.hashes.p});
}

// 7. to the host (the caller DEFLATEs the large ones)
inline void Engine::copyEncodeOutput(EncodeCall& e, std::string& out, std::vector<u64>& offs, std::string& hashesOut) {
  const size_t n = e.n;
  out.resize(e.total); offs.assign(n + 1, 0); hashesOut.resize(n * 32);
  if (!n) return;
  if (e.total) d2h(ctx, &out[0], e.out.p, e.total);
  d2h(ctx, offs.data(), e.outOff.p, (n + 1) * 8); d2h(ctx, &hashesOut[0], e.hashes.p, n * 32); sync(ctx);
}

// The first failing change (firstFailingChange), and for it the error of its earliest phase
inline void Engine::throwEncodeError(EncodeCall& e, const u64* w) {
  const auto [best, phase] = firstFailingChange(w, EP_NUM, EP_OPS, e.opBase.p, e.n);
  encodeFailed = best; const u32 code = (u32)(w[phase] & 0xff);
  const std::string at = "change table: change " + std::to_string(best) + ": ";
  switch (code) {
    case EE_CHG_OPS: throw Error(AMG_ERR_RANGE, at + "ops out of range");
    case EE_CHG_PREDS: throw Error(AMG_ERR_RANGE, at + "preds out of range");
    case EE_CHG_ACTORS: throw Error(AMG_ERR_RANGE, at + "actor table out of range");
    case EE_ACTOR_ENTRY: throw Error(AMG_ERR_RANGE, at + "actor id out of range");
    case EE_CHG_MSG: throw Error(AMG_ERR_RANGE, at + "message out of range");
    case EE_CHG_DEPS: throw Error(AMG_ERR_RANGE, at + "deps out of range");
    case EE_CHG_EXTRA: throw Error(AMG_ERR_RANGE, at + "extra bytes out of range");
    case EE_NUM_RANGE: throw Error(AMG_ERR_RANGE, "number out of range");
    case EE_TOO_LARGE: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: more than 2^31 preds in one change");
    case EE_CHANGE_SIZE: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change " + std::to_string(best) + " may encode to 4 GiB or more (its ops' key and value bytes are counted once per op)");
    case EE_OP_KEYSTR: throw Error(AMG_ERR_RANGE, at + "key string out of range");
    case EE_OP_VALUE: throw Error(AMG_ERR_RANGE, at + "value out of range");
    case EE_OP_PREDS: throw Error(AMG_ERR_RANGE, at + "op preds out of range");
    case EE_OBJ: throw Error(AMG_ERR_RANGE, "Unexpected objectId reference");
    case EE_KEY: throw Error(AMG_ERR_RANGE, "Unexpected operation key");
    case EE_ACTION: throw Error(AMG_ERR_RANGE, "Unexpected operation action");
    default: break;
  }
  if (phase == EP_OPS) {   // the messages that name a value of the op
    const size_t j = (size_t)(w[phase] >> 8); ChangeRec r; u32 opBase = 0; d2h(ctx, &r, e.T.ch + best, sizeof(r)); d2h(ctx, &opBase, e.opBase.p + best, 4); sync(ctx);
    OpRec o; d2h(ctx, &o, e.T.ops + r.firstOp + (j - opBase), sizeof(o)); sync(ctx);
    auto actorIndex = [](u32 a) { return "No actor index " + std::to_string(a); };
    switch (code) {
      case EE_KEY_ACTOR: throw Error(AMG_ERR_RANGE, actorIndex(o.keyActor));
      case EE_CHLD_ACTOR: throw Error(AMG_ERR_RANGE, actorIndex(o.chldActor));
      case EE_CHLD_NULL: throw Error(AMG_ERR_RANGE, "Mismatched child columns: " + std::to_string(o.chldCtr) + " and None");
      case EE_PRED_NULL: throw Error(AMG_ERR_RANGE, "Not a valid opId: a pred counter is null");
      case EE_PRED_ACTOR: {
        std::vector<u32> pr(2 * (size_t)o.predNum + 2); d2h(ctx, pr.data(), e.T.preds + 2 * (size_t)o.predFirst, (size_t)o.predNum * 8); sync(ctx);
        for (u32 k = 0; k < o.predNum; k++) if (pr[2 * k] >= r.nActors) throw Error(AMG_ERR_RANGE, actorIndex(pr[2 * k]));
        break;
      }
      case KE_FLOAT_LEN: throw Error(AMG_ERR_RANGE, "Invalid length for floating point number: " + std::to_string(o.valLen >> 4));
      default: break;
    }
  }
  throwKernelError(w[phase]);
}

inline void Engine::gatherHashes(const std::vector<u32>& idx, std::string& out) {
  out.assign(idx.size() * 32, '\0');
  if (idx.empty()) return;
  spans.resume(SPAN_SYNC);
  syncIdx.ensure(ctx, idx.size() + 1); h2d(ctx, syncIdx.p, idx.data(), idx.size() * 4);
  syncHashOut.ensure(ctx, idx.size() * 32);
  foreach(ctx, idx.size(), SyncHashGatherKernel{hashes.p, syncIdx.p, syncHashOut.p});
  d2h(ctx, &out[0], syncHashOut.p, out.size()); sync(ctx);
  spans.stop();   // adds to the span of the syncChangesToSend call it follows
}


// ------------------------------------------------------------ getHistory snapshots (snapshot.cuh; src/automerge.js:105-118)
// out[i] = the flat whole-document patch that getPatch(loadChanges(init(), getAllChanges()[0, prefixLens[i]))) returns
inline void Engine::historyPatches(const u64* prefixLens, size_t n, std::vector<std::string>& out) {
  out.clear(); spans.ms[SPAN_HISTORY] = 0;   // also when the call fails before its span starts
  for (size_t i = 0; i < n; i++)
    if (prefixLens[i] > numApplied) throw Error(AMG_ERR_RANGE, "history prefix length " + std::to_string(prefixLens[i]) + " exceeds the " + std::to_string(numApplied) + " applied changes");
  if (n == 0) return;
  computeHashGraph();   // the prefixes' heads are change hashes (as amg_decode_history)
  HistoryPatchCall h; h.C = numApplied; h.A = st.actorIds.size(); h.N = numRows; h.S = numSucc;
  if (h.C >= (1u << 31) || h.N + h.S >= (1u << 31)) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: document too large for history snapshots");
  struct SideJoin { Ctx& c; ~SideJoin() { side_join(c); } } sideJoin{ctx};
  spans.start(SPAN_HISTORY);
  clearErr();
  if (h.C) { snapChangeMeta(h); snapActorOrder(h); snapChangeIndexes(h); }
  const Ord ord{actorRank.p, bits_for(std::max<size_t>(h.A, 2) - 1)};
  for (size_t i = 0; i < n; i++) {
    const size_t k = (size_t)prefixLens[i];
    clearErr();
    const size_t Nk = snapFilter(h, k);
    PatchOut p;
    buildPatch(PatchInputs{snapDoc.view(), Nk, true, snapSuccOff.p, snapSucc.p, snapSuccCnt.p, ord}, p);
    side_join(ctx); sync(ctx);
    checkErr();
    snapHeader(h, k, p);
    finishPatch(p);
    out.emplace_back((const char*)p.bytes, p.bytesLen);   // patchBuf is reused by the next prefix length
  }
  spans.stop();
}

// 1. actor number, seq, maxOp and dependency indexes of every applied change (the change metadata phase save() uses)
inline void Engine::snapChangeMeta(HistoryPatchCall& h) {
  const size_t C = h.C;
  h.m = ChangeMetaCall{C, loaded.numChanges, C - loaded.numChanges};
  parseChangeMeta(h.m);
  h.D = (size_t)h.m.loadedDeps + h.m.laterDeps;
  for (DBuf<long long>* b : {&h.cActor, &h.cSeq, &h.cMaxOp, &h.cDepsNum}) b->ensure(ctx, C + 1);
  h.strOff.ensure(ctx, std::max(C, h.D) + 1); h.strLen.ensure(ctx, std::max(C, h.D) + 1); h.depsNum32.ensure(ctx, C + 1); h.depBase.ensure(ctx, C + 2);
  h.depIdxV.ensure(ctx, h.D + 1); h.depIdx.ensure(ctx, h.D + 1);
  changeMetaColumn(h.m, CC_ACTOR, h.cActor.p, h.strOff.p, h.strLen.p);
  changeMetaColumn(h.m, CC_SEQ, h.cSeq.p, h.strOff.p, h.strLen.p);
  changeMetaColumn(h.m, CC_MAX_OP, h.cMaxOp.p, h.strOff.p, h.strLen.p);
  changeMetaColumn(h.m, CC_DEPS_NUM, h.cDepsNum.p, h.strOff.p, h.strLen.p);
  changeMetaColumn(h.m, CC_DEPS_INDEX, h.depIdxV.p, h.strOff.p, h.strLen.p);
  foreach(ctx, C, HistI64ToU32Kernel{h.cDepsNum.p, h.depsNum32.p});
  scan_exclusive(ctx, scanTmp, h.depsNum32.p, h.depBase.p, C);
  foreach(ctx, h.D, HistI64ToU32Kernel{h.depIdxV.p, h.depIdx.p});
  checkErr();
}

// 2. each actor's changes by seq (the history kernels: key = actor << 40 | seq, radix sort, segment starts)
inline void Engine::snapActorOrder(HistoryPatchCall& h) {
  const size_t C = h.C, A = h.A;
  h.chKey.ensure(ctx, C + 1); h.changeOrder.ensure(ctx, C + 1); h.actorStart.ensure(ctx, A + 2);
  foreach(ctx, C, HistChangeKeyKernel{h.cActor.p, h.cSeq.p, h.chKey.p, h.changeOrder.p});
  radix_sort_pairs(ctx, sortTmp, h.chKey, h.changeOrder, C, 0, 40); radix_sort_pairs(ctx, sortTmp, h.chKey, h.changeOrder, C, 40, 57);
  foreach(ctx, A + 1, HistLowerBoundKernel{h.chKey.p, (u32)C, 40, h.actorStart.p});
}

// 3. the change of every row id and succ entry; the first dependent of every change
inline void Engine::snapChangeIndexes(HistoryPatchCall& h) {
  const size_t C = h.C, N = h.N, S = h.S;
  h.rowChange.ensure(ctx, N + 1); h.succChange.ensure(ctx, S + 1); h.firstDep.ensure(ctx, C + 1);
  foreach(ctx, N, SnapChangeOfKernel{doc.id.p, h.actorStart.p, h.changeOrder.p, h.cMaxOp.p, (u32)h.A, h.rowChange.p, errWord.p});
  foreach(ctx, S, SnapChangeOfKernel{succ.p, h.actorStart.p, h.changeOrder.p, h.cMaxOp.p, (u32)h.A, h.succChange.p, errWord.p});
  dev_memset(ctx, h.firstDep.p, 0xff, (C + 1) * 4);
  foreach(ctx, h.D, SnapFirstDepKernel{h.depBase.p, h.depIdx.p, (u32)C, h.firstDep.p});
  checkErr();
}

// 4. per prefix length: flag the kept rows and count their kept succ entries, two scans, one gather
inline size_t Engine::snapFilter(HistoryPatchCall& h, size_t k) {
  const size_t N = h.N;
  if (k == 0 || N == 0) return 0;
  for (DBuf<u32>* b : {&h.keep, &h.cnt}) b->ensure(ctx, N + 1);
  for (DBuf<u32>* b : {&h.rowPos, &h.cntPos}) b->ensure(ctx, N + 2);
  foreach(ctx, N, SnapKeepKernel{h.rowChange.p, succOff.p, h.succChange.p, (u32)k, h.keep.p, h.cnt.p});
  scan_exclusive(ctx, scanTmp, h.keep.p, h.rowPos.p, N);
  scan_exclusive(ctx, scanTmp, h.cnt.p, h.cntPos.p, N);
  u32 Nk = 0, Sk = 0; readU32x2(h.rowPos.p + N, h.cntPos.p + N, &Nk, &Sk);
  snapDoc.ensure(ctx, (size_t)Nk + 1); snapSuccOff.ensure(ctx, (size_t)Nk + 2); snapSuccCnt.ensure(ctx, (size_t)Nk + 2); snapSucc.ensure(ctx, (size_t)Sk + 1);
  foreach(ctx, N, SnapGatherKernel{doc.view(), succOff.p, succ.p, h.succChange.p, (u32)k, (u32)N, h.keep.p, h.rowPos.p, h.cntPos.p,
                                   snapDoc.view(), snapSuccOff.p, snapSucc.p, snapSuccCnt.p});
  return Nk;
}

// 5. per prefix length: heads (changes whose first dependent is not in the prefix, sorted by hash), clock and maxOp
inline void Engine::snapHeader(HistoryPatchCall& h, size_t k, PatchOut& out) {
  const size_t A = h.A;
  out.pendingChanges = 0; out.actors = st.actorIds; out.maxOp = 0; out.clock.clear(); out.deps.clear();
  if (k == 0) return;
  h.headFlag.ensure(ctx, k + 1); h.headPos.ensure(ctx, k + 2); h.headIdx.ensure(ctx, k + 1); h.clock.ensure(ctx, A + 2);
  dev_memset(ctx, h.clock.p, 0, (A + 1) * 8);   // [A]: maxOp
  foreach(ctx, k, SnapHeaderKernel{h.cActor.p, h.cSeq.p, h.cMaxOp.p, h.firstDep.p, (u32)k, (u32)A, h.headFlag.p,
                                   reinterpret_cast<unsigned long long*>(h.clock.p), reinterpret_cast<unsigned long long*>(h.clock.p + A)});
  scan_exclusive(ctx, scanTmp, h.headFlag.p, h.headPos.p, k);
  foreach(ctx, k, CompactKernel{h.headFlag.p, h.headPos.p, h.headIdx.p});
  const u32 nh = readU32(h.headPos.p + k);
  h.headHashes.ensure(ctx, (size_t)nh * 32 + 32);
  foreach(ctx, nh, SyncHashGatherKernel{hashes.p, h.headIdx.p, h.headHashes.p});
  std::vector<u64> clock(A + 1); std::vector<std::array<u8, 32>> heads(nh);
  d2h(ctx, clock.data(), h.clock.p, (A + 1) * 8);
  if (nh) d2h(ctx, heads.data(), h.headHashes.p, (size_t)nh * 32);
  sync(ctx);
  std::sort(heads.begin(), heads.end());
  out.maxOp = clock[A]; out.deps = std::move(heads);
  for (size_t a = 0; a < A; a++) if (clock[a] > 0) out.clock.emplace_back((u32)a, clock[a]);
}

// ------------------------------------------------------------ merge (merge.cuh; new.js:1979-1997, src/automerge.js:61-67)
// Which changes: every applied change of src whose hash this document has not applied, one table lookup each. That is
// exactly the set the reference's walk from src's heads visits (DESIGN.md section 3): a document applies a change only
// after its dependencies, so every ancestor of a change this document has is here as well, and every absent change is
// reached from src's heads through absent changes only. The order is the walk's; it runs on the host over the absent
// changes' dependency indexes, for the reason syncChangesToSend gives (a device walk needs one launch per level).
inline void Engine::changesAddedFrom(Engine& src, std::vector<u32>& order) {
  order.clear();
  computeHashGraph();   // new.js:1980; the package builds both documents' graphs (DESIGN.md section 5)
  src.computeHashGraph();
  if (src.ctx.device != ctx.device)
    throw Error(AMG_ERR_UNSUPPORTED, "amgpu: the documents are on different devices (" + std::to_string(src.ctx.device) + ", " + std::to_string(ctx.device) + ")");
  sync(src.ctx);   // src's buffers are read on this engine's stream
  const size_t C = src.numApplied;
  if (C == 0) return;
  clearErr();
  // 1. presence: this document's hashes in a table, one probe per change of src, then flag -> scan -> compact
  const u64 ownMask = hashTableOf(hashes.p, numApplied);
  mergeAbsent.ensure(ctx, C + 1); mergeSlot.ensure(ctx, C + 2);
  foreach(ctx, C, MergeProbeKernel{hashes.p, hashTable.p, ownMask, src.hashes.p, mergeAbsent.p});
  scan_exclusive(ctx, scanTmp, mergeAbsent.p, mergeSlot.p, C);
  const size_t K = readU32(mergeSlot.p + C);
  if (K == 0) return;
  mergeList.ensure(ctx, K + 1);
  foreach(ctx, C, CompactKernel{mergeAbsent.p, mergeSlot.p, mergeList.p});
  std::vector<u32> absent(K); d2h(ctx, absent.data(), mergeList.p, K * 4); sync(ctx);
  // 2. the absent changes' dependencies in header order (the order of dependenciesByHash) and src's heads, as change
  //    indexes of src: their headers in src's arena, resolved against src's hashes (parseChangeHeaders, resolveChangeDeps)
  std::vector<HostChange> pairs(K); for (size_t k = 0; k < K; k++) pairs[k] = src.changes[absent[k]];
  const u32 D = parseChangeHeaders(src.arena.p, pairs.data(), K);
  checkErr();
  const u64 srcMask = resolveChangeDeps(src.arena.p, src.hashes.p, C, K, 0, D);
  const size_t H = src.st.heads.size();
  mergeHeads.ensure(ctx, H * 32 + 32); mergeHeadIdx.ensure(ctx, H + 1);
  std::vector<u8> headBytes(H * 32); for (size_t i = 0; i < H; i++) memcpy(headBytes.data() + 32 * i, src.st.heads[i].data(), 32);
  h2d(ctx, mergeHeads.p, headBytes.data(), H * 32);
  foreach(ctx, H, HashLookupKernel{src.hashes.p, hashTable.p, srcMask, mergeHeads.p, mergeHeadIdx.p});
  std::vector<u32> base(K + 1), deps(D), stack(H);
  d2h(ctx, base.data(), depBase.p, (K + 1) * 4); d2h(ctx, deps.data(), depIdx.p, (size_t)D * 4); d2h(ctx, stack.data(), mergeHeadIdx.p, H * 4); sync(ctx);
  // 3. new.js:1983-1994: heads in order, popped from the back; the seen test at pop time; dependencies pushed in header
  //    order; a change this document has stops the walk. Then reversed (:1996).
  std::vector<u32> posOf(C, EMPTY32); for (size_t k = 0; k < K; k++) posOf[absent[k]] = (u32)k;
  std::vector<u8> seen(K, 0);
  while (!stack.empty()) {
    const u32 c = stack.back(); stack.pop_back();
    const u32 k = c < C ? posOf[c] : EMPTY32;
    if (k == EMPTY32 || seen[k]) continue;
    seen[k] = 1; order.push_back(c);
    stack.insert(stack.end(), deps.begin() + base[k], deps.begin() + base[k + 1]);
  }
  std::reverse(order.begin(), order.end());
}

// The changes to send are the bytes getChangesAdded returns (amg_backend::changeBytes): a change's DEFLATEd original when
// it has one, else its plain bytes. A change getChangesAdded would DEFLATE on the way out (exportsDeflated) goes over
// plain and marked instead, so that this document hands it out DEFLATEd later, as if it had received it that way.
inline void Engine::mergeFrom(Engine& src, bool wantPatch, PatchOut& out) {
  spans.start(SPAN_MERGE);
  std::vector<u32> idx; changesAddedFrom(src, idx);
  const size_t K = idx.size();
  std::vector<u64> offs(K + 1, 0); std::vector<MergeRange> ranges(K); std::vector<u8> marks(K + 1, 0);
  for (size_t k = 0; k < K; k++) {
    const u32 c = idx[k]; const HostChange* o = src.originalOf(c); const HostChange r = o ? *o : src.changes[c];
    marks[k] = src.exportsDeflated(c) ? 1 : 0;
    ranges[k] = MergeRange{offs[k], r.off, r.len}; offs[k + 1] = offs[k] + r.len;
  }
  if ((u64)arenaLen + offs[K] + 64 >= 0xfff00000ULL) throw Error(AMG_ERR_UNSUPPORTED, "amgpu: change arena limited to 4 GiB per document");
  mergeBlob.ensure(ctx, offs[K] + 64); mergeRanges.ensure(ctx, K + 1);
  h2d(ctx, mergeRanges.p, ranges.data(), K * sizeof(MergeRange));
  merge_gather(ctx, K, MergeGatherKernel{src.arena.p, mergeBlob.p, mergeRanges.p});
  applyChanges(nullptr, nullptr, K, mergeBlob.p, offs.data(), false, wantPatch, out, marks.data());   // the device-blob path of amg_apply_changes_packed
  spans.stop();
}

// ------------------------------------------------------------ applyLocalChange (backend.js:54-91)
// The checks and the previous hash come from the engine's clock, lastChange and hashes: no host hash graph. The change
// bytes go from the encoder's output to the apply's arena without leaving the device.
inline void Engine::applyLocalChange(const u8* table, size_t len, bool wantPatch, PatchOut& out, std::string& binary) {
  spans.start(SPAN_LOCAL);
  EncodeCall e; e.len = len; encodeFailed = 0;
  clearErr();
  stageEncodeInput(e, table);
  if (e.n != 1) throw Error(AMG_ERR_RANGE, "change table: applyLocalChange takes one change request, not " + std::to_string(e.n));
  // 1. the author (actor entry 0) and seq. A record without a readable author skips the checks: validateTable reports it.
  ChangeRec r; d2h(ctx, &r, e.T.ch, sizeof(r)); sync(ctx);
  std::string author; bool haveAuthor = false;
  if (r.nActors > 0 && r.actorFirst < e.T.nActors) {
    ActorRef ar; d2h(ctx, &ar, e.T.actors + r.actorFirst, sizeof(ar)); sync(ctx);
    if (e.T.inside(ar.off, ar.len)) { author.resize(ar.len); d2h(ctx, &author[0], e.T.t + ar.off, ar.len); sync(ctx); haveAuthor = true; }
  }
  auto actorNum = [&]() { return (size_t)(std::find(st.actorIds.begin(), st.actorIds.end(), author) - st.actorIds.begin()); };
  auto unknownChange = [&](u64 seq) { return Error(AMG_ERR_RANGE, "Unknown change: actorId = " + hex_of((const u8*)author.data(), author.size()) + ", seq = " + std::to_string(seq)); };
  if (haveAuthor) {
    const size_t a = actorNum(); const u64 clock = a < st.actorIds.size() ? st.clock[a] : 0;
    if (r.seq <= clock) throw Error(AMG_ERR_RANGE, "Change request has already been applied");
    if (r.seq > 1) {   // 2. the author's change seq - 1 is its last applied change
      if (r.seq - 1 > clock) throw unknownChange(r.seq - 1);
      if (!loaded.haveHashGraph) {   // a loaded document knows the hashes of its heads only (new.js:1721-1725)
        const u32 idx = readU32(lastChange.p + a);
        if (idx < loaded.numChanges && std::find(st.headIdx.begin(), st.headIdx.end(), idx) == st.headIdx.end()) computeHashGraph();
      }
      e.T.prevHashes = hashes.p; e.T.prevIdx = lastChange.p + a;
    }
  }
  // 3. encoded, the previous hash added to the deps by EncHashKernel
  validateTable(e); encodeActorTables(e); encodePrep(e); encodeColumns(e); encodeHashes(e);
  // 4. applied from device memory; a change that encodeChange returns DEFLATEd goes out DEFLATEd, as after the host route
  const u64 offs[2] = {0, e.total}; const u8 mark[1] = {(u8)(e.total >= 256 ? 1 : 0)};
  applyChanges(nullptr, nullptr, 1, e.out.p, offs, true, wantPatch, out, mark);
  binary.resize(e.total); std::array<u8, 32> hash;
  d2h(ctx, &binary[0], e.out.p, e.total); d2h(ctx, hash.data(), e.hashes.p, 32); sync(ctx);
  { const size_t a = actorNum(); if (a == st.actorIds.size() || st.clock[a] < r.seq) throw unknownChange(r.seq); }   // it waits in the queue (backend.js:84)
  // 5. the patch without the new change's own hash (backend.js:86-88)
  out.deps.erase(std::remove(out.deps.begin(), out.deps.end(), hash), out.deps.end());
  finishPatch(out);
  spans.stop();
}

// ------------------------------------------------------------ hash-graph queries (graph.cuh; new.js:1921-2028)
// The dependents lists are appended on the host: the graph grows batch by batch, and the walks that read it run on the
// host anyway, so the integers come back once. A device scatter into one CSR would rebuild it whole for every batch.
inline void Engine::ChangeGraph::add(u32 c, const u32* dep, size_t nDep, u32 actor, const u8* h) {
  for (size_t j = 0; j < nDep; j++) {
    const u32 d = dep[j];   // an applied change's dependencies were applied before it
    if (d >= c) throw Error(AMG_ERR_INTERNAL, "amgpu: change " + std::to_string(c) + " depends on a change that is not applied before it");
    const u32 k = (u32)deps.size();
    deps.push_back(d); depOwner.push_back(c); nextDependent.push_back(EMPTY32);
    if (firstDependent[d] == EMPTY32) firstDependent[d] = k; else nextDependent[lastDependent[d]] = k;
    lastDependent[d] = k;
  }
  depBase.push_back((u32)deps.size()); firstDependent.push_back(EMPTY32); lastDependent.push_back(EMPTY32);
  if (byActor.size() <= actor) byActor.resize((size_t)actor + 1);
  byActor[actor].push_back(c);
  hash.emplace_back(); memcpy(hash.back().data(), h, 32);
  auto insert = [&](u32 i) { u64 key; memcpy(&key, hash[i].data(), 8); u64 s = mix64(key) & (slots.size() - 1); while (slots[s] != EMPTY32) s = (s + 1) & (slots.size() - 1); slots[s] = i; };
  if (2 * hash.size() > slots.size()) {   // keep the table at most half full
    slots.assign(pow2_at_least(std::max<size_t>(64, 4 * hash.size())), EMPTY32);
    for (u32 i = 0; i < (u32)hash.size(); i++) insert(i);
  } else insert(c);
  known = (size_t)c + 1;
}
inline u32 Engine::ChangeGraph::find(const u8* h) const {
  if (slots.empty()) return DEP_MISSING;
  u64 key; memcpy(&key, h, 8);
  for (u64 s = mix64(key) & (slots.size() - 1); slots[s] != EMPTY32; s = (s + 1) & (slots.size() - 1))
    if (memcmp(hash[slots[s]].data(), h, 32) == 0) return slots[s];
  return DEP_MISSING;
}

// commit: the batch's gate tables, copied device to device behind the ones kept before (read back by the next query)
inline void Engine::keepGraphInputs(ApplyCall& a) {
  GraphInputs& k = graphInputs; const size_t B = a.B, D = a.D;
  GraphInputs::Batch b{numApplied, B, D, a.numNew, k.usedB, k.usedBase, k.usedD};
  k.applied.ensure(ctx, b.offB + B + 1, b.offB); k.rank.ensure(ctx, b.offB + B + 1, b.offB); k.actor.ensure(ctx, b.offB + B + 1, b.offB);
  k.depBase.ensure(ctx, b.offBase + B + 2, b.offBase); k.depIdx.ensure(ctx, b.offD + D + 1, b.offD);
  d2d(ctx, k.applied.p + b.offB, applied.p, B); d2d(ctx, k.rank.p + b.offB, appRank.p, B * 4); d2d(ctx, k.actor.p + b.offB, changeActor.p, B * 4);
  d2d(ctx, k.depBase.p + b.offBase, depBase.p, (B + 1) * 4); d2d(ctx, k.depIdx.p + b.offD, depIdx.p, D * 4);
  k.usedB += B; k.usedBase += B + 1; k.usedD += D; k.batches.push_back(b);
}

inline void Engine::graphFromBatch(const GraphInputs::Batch& b) {
  GraphInputs& k = graphInputs; const size_t B = b.B;
  std::vector<u8> ap(B + 1); std::vector<u32> rank(B + 1), actor(B + 1), base(B + 2), dep(b.D + 1); std::vector<std::array<u8, 32>> hs(b.numNew);
  d2h(ctx, ap.data(), k.applied.p + b.offB, B); d2h(ctx, rank.data(), k.rank.p + b.offB, B * 4); d2h(ctx, actor.data(), k.actor.p + b.offB, B * 4);
  d2h(ctx, base.data(), k.depBase.p + b.offBase, (B + 1) * 4); d2h(ctx, dep.data(), k.depIdx.p + b.offD, b.D * 4);
  d2h(ctx, hs.data(), hashes.p + b.first * 32, b.numNew * 32); sync(ctx);
  std::vector<u32> byRank(b.numNew, EMPTY32);
  for (size_t e = 0; e < B; e++) if (ap[e]) byRank[rank[e]] = (u32)e;
  std::vector<u32> ds;
  for (size_t r = 0; r < b.numNew; r++) {
    const u32 e = byRank[r];
    if (e == EMPTY32) throw Error(AMG_ERR_INTERNAL, "amgpu: change graph: an application rank without its change");
    ds.clear();
    for (u32 j = base[e]; j < base[e + 1]; j++) {   // gate numbering -> application index
      const u32 d = dep[j];
      ds.push_back(d == DEP_MISSING || d < b.first ? d : (d - (u32)b.first < B && ap[d - b.first] ? (u32)b.first + rank[d - b.first] : DEP_MISSING));
    }
    graph.add((u32)(b.first + r), ds.data(), ds.size(), actor[e], hs[r].data());
  }
}

inline void Engine::graphFromHeaders(size_t from, size_t to) {
  const size_t K = to - from;
  clearErr();
  const u32 D = parseChangeHeaders(arena.p, changes.data() + from, K);
  checkErr();
  resolveChangeDeps(arena.p, hashes.p, to, K, from, D);
  graphVals.ensure(ctx, K + 1);
  foreach(ctx, K, SaveChangeValKernel{SM_ACTOR, arena.p, meta.p, actorSlots.p, (u64)actorCap - 1, graphVals.p, nullptr, nullptr, errWord.p});
  std::vector<u32> base(K + 1), deps((size_t)D + 1); std::vector<long long> actor(K); std::vector<std::array<u8, 32>> hs(K);
  d2h(ctx, base.data(), depBase.p, (K + 1) * 4); d2h(ctx, deps.data(), depIdx.p, (size_t)D * 4); d2h(ctx, actor.data(), graphVals.p, K * 8);
  d2h(ctx, hs.data(), hashes.p + from * 32, K * 32); sync(ctx);
  checkErr();
  for (size_t b = 0; b < K; b++) graph.add((u32)(from + b), deps.data() + base[b], base[b + 1] - base[b], (u32)actor[b], hs[b].data());
}

// Brings the graph up to [0, numApplied): kept batches where they continue it, header parses for the rest
inline void Engine::extendGraph() {
  GraphInputs& k = graphInputs;
  size_t next = 0;
  while (graph.known < numApplied) {
    while (next < k.batches.size() && k.batches[next].first < graph.known) next++;   // already in the graph
    if (next < k.batches.size() && k.batches[next].first == graph.known) { graphFromBatch(k.batches[next++]); continue; }
    graphFromHeaders(graph.known, next < k.batches.size() ? k.batches[next].first : numApplied);
  }
  k.clear();
}

inline void Engine::lookupQueries(size_t n, size_t count, std::vector<u32>& idx) {
  idx.assign(n, DEP_MISSING);
  if (n == 0 || count == 0) return;
  graphIdx.ensure(ctx, n + 1);
  const u64 mask = hashTableOf(hashes.p, count);
  foreach(ctx, n, HashLookupKernel{hashes.p, hashTable.p, mask, graphQueries.p, graphIdx.p});
  d2h(ctx, idx.data(), graphIdx.p, n * 4); sync(ctx);
}

inline void Engine::lookupHashes(const u8* hs, size_t n, std::vector<u32>& idx) {
  graphQueries.ensure(ctx, n * 32 + 32);
  if (n) h2d(ctx, graphQueries.p, hs, n * 32);
  lookupQueries(n, numApplied, idx);
}

// new.js:1921-1973. haveDeps and the heads are looked up in the graph's hashes; an unknown hash raises before any traversal. The
// fast path walks forward from haveDeps through the dependents (no seen test at pop: a change reached from two seen parents
// is returned twice, as in the reference); when it gives up, the slow path returns every change that is not an ancestor of
// haveDeps, in application order.
inline void Engine::changesSince(const u8* haveDeps, size_t n, std::vector<u32>& out) {
  out.clear();
  computeHashGraph();
  spans.start(SPAN_GRAPH);
  if (n == 0) { out.resize(changes.size()); for (size_t i = 0; i < out.size(); i++) out[i] = (u32)i; spans.stop(); return; }
  extendGraph();
  spans.stop();
  const size_t H = st.heads.size();
  std::vector<u32> idx(n + H);   // haveDeps, then the heads
  for (size_t i = 0; i < n; i++) idx[i] = graph.find(haveDeps + 32 * i);
  for (size_t h = 0; h < H; h++) idx[n + h] = graph.find(st.heads[h].data());
  for (size_t i = 0; i < n; i++) if (idx[i] == DEP_MISSING) throw Error(AMG_ERR_RANGE, "hash not found: " + hex_of(haveDeps + 32 * i, 32));
  const ChangeGraph& g = graph;
  std::vector<u8> seen(numApplied, 0); std::vector<u32> stack;
  auto push = [&](u32 c) { stack.push_back(c); };
  for (size_t i = 0; i < n; i++) { seen[idx[i]] = 1; g.eachDependent(idx[i], push); }
  // Reference quirk reproduced on purpose (new.js:1938-1955): the traversal stops at a change with an unseen dependency, but
  // the test below only looks at the stack and the heads - when that change was the last one on the stack and the heads
  // have all been seen, the fast path still answers, without the changes that are concurrent to `haveDeps`.
  while (!stack.empty()) {
    const u32 c = stack.back(); stack.pop_back(); seen[c] = 1; out.push_back(c);
    bool all = true;
    for (u32 k = g.depBase[c]; k < g.depBase[c + 1] && all; k++) all = seen[g.deps[k]] != 0;
    if (!all) break;
    g.eachDependent(c, push);
  }
  bool headsSeen = true;
  for (size_t h = 0; h < H; h++) if (idx[n + h] == DEP_MISSING || !seen[idx[n + h]]) headsSeen = false;
  if (stack.empty() && headsSeen) return;
  out.clear(); std::fill(seen.begin(), seen.end(), 0);
  stack.assign(idx.begin(), idx.begin() + n);
  while (!stack.empty()) {
    const u32 c = stack.back(); stack.pop_back();
    if (seen[c]) continue;
    seen[c] = 1; stack.insert(stack.end(), g.deps.begin() + g.depBase[c], g.deps.begin() + g.depBase[c + 1]);
  }
  for (size_t i = 0; i < changes.size(); i++) if (!seen[i]) out.push_back((u32)i);
}

// new.js:1999-2002: one lookup among the applied changes (a queued change has no index yet)
inline bool Engine::changeIndexOf(const u8* hash, u32& idx) {
  computeHashGraph();
  spans.start(SPAN_GRAPH);
  std::vector<u32> found; lookupHashes(hash, 1, found);
  spans.stop();
  idx = found[0];
  return idx != DEP_MISSING;
}

// new.js:2014-2028. The queued changes' headers are parsed and their hashes computed on the device (SHA-256 over bytes
// [8, len) of the inflated change, written behind the applied hashes); their dependencies and the given heads are looked up
// in one table over the applied and the queued hashes. Whatever is in neither is missing.
inline void Engine::missingDeps(const u8* heads, size_t n, std::vector<std::array<u8, 32>>& out) {
  out.clear();
  computeHashGraph();
  spans.start(SPAN_GRAPH);
  const size_t C = numApplied, Q = queue.size();
  u32 D = 0;
  clearErr();
  if (Q > 0) {
    D = parseChangeHeaders(arena.p, queue.data(), Q);
    checkErr();
    hashes.ensure(ctx, (C + Q) * 32 + 64, C * 32);
    foreach(ctx, Q, ShaKernel{arena.p, chOff.p, chLen.p, hashes.p + C * 32, errWord.p, nullptr, nullptr});
  }
  graphQueries.ensure(ctx, ((size_t)D + n) * 32 + 32);
  if (D > 0) foreach(ctx, Q, DepHashCopyKernel{arena.p, meta.p, depBase.p, graphQueries.p});
  if (n > 0) h2d(ctx, graphQueries.p + (size_t)D * 32, heads, n * 32);
  std::vector<u32> idx; lookupQueries((size_t)D + n, C + Q, idx);
  std::vector<std::array<u8, 32>> deps(D);
  if (D > 0) { d2h(ctx, deps.data(), graphQueries.p, (size_t)D * 32); sync(ctx); }
  checkErr();
  spans.stop();
  for (size_t i = 0; i < (size_t)D + n; i++) {
    if (idx[i] != DEP_MISSING) continue;
    if (i < D) out.push_back(deps[i]);
    else { out.emplace_back(); memcpy(out.back().data(), heads + (i - D) * 32, 32); }
  }
  std::sort(out.begin(), out.end());
  out.erase(std::unique(out.begin(), out.end()), out.end());
}

// hashesByActor[actor][index] (the host-side applyLocalChange's previous hash, backend.js:54-91)
inline bool Engine::hashByActor(const std::string& actor, u64 index, u8* out) {
  computeHashGraph();
  spans.start(SPAN_GRAPH);
  extendGraph();
  const size_t a = (size_t)(std::find(st.actorIds.begin(), st.actorIds.end(), actor) - st.actorIds.begin());
  const bool found = a < graph.byActor.size() && index < graph.byActor[a].size();
  if (found) memcpy(out, graph.hash[graph.byActor[a][index]].data(), 32);
  spans.stop();
  return found;
}

}  // namespace amg
