// amgpu — host orchestration of the change-replay pipeline (one Engine = one backend document).
//
// Mirrors class BackendDoc (reference backend/new.js:1694-2069): applyChanges (:1797-1879) and
// getPatch (:2060-2068) run as sequences of CUDA kernels over device-resident state:
//   arena   : every applied / queued change's bytes back to back (values and keys are referenced in place)
//   hashes  : SHA-256 of every applied change                      (gate)
//   doc     : document rows in document order, SoA, + succ CSR      (op set)
//   actors  : byte-string table of actor ids -> document actor index
// An applyChanges call is atomic (reference :1793-1795): all kernels write into scratch buffers; the
// persistent state is swapped in only after the last error check passed.
#pragma once
#include <algorithm>
#include <array>
#include <initializer_list>
#include <map>
#include <memory>
#include <thread>
#include <chrono>
#include <zlib.h>
#ifndef AMG_EMU
#include <nvtx3/nvToolsExt.h>
#endif
#include "patch.cuh"
#include "inflate.cuh"
#include "encode.cuh"
#include "prims.cuh"
#include "domlocal.cuh"
#include "doccols.cuh"
#include "history.cuh"
#include "sync.cuh"
#include "changes.cuh"
#include "encchg.cuh"
#include "snapshot.cuh"
#include "merge.cuh"
#include "graph.cuh"
#include "unknowncols.hpp"

namespace amg {

struct DocBufs {
  DBuf<u64> id, obj, key; DBuf<u32> keyStrOff, keyStrLen, flags, valLen, valOff, time;
  template <class F> void each(DocBufs& o, F f) { f(id, o.id); f(obj, o.obj); f(key, o.key); f(keyStrOff, o.keyStrOff); f(keyStrLen, o.keyStrLen); f(flags, o.flags); f(valLen, o.valLen); f(valOff, o.valOff); f(time, o.time); }
  void ensure(Ctx& c, size_t n, size_t keep = 0) { each(*this, [&](auto& x, auto&) { x.ensure(c, n, keep); }); }
  DocRows view() { return DocRows{id.p, obj.p, key.p, keyStrOff.p, keyStrLen.p, flags.p, valLen.p, valOff.p, time.p}; }
  void swap(DocBufs& o) { each(o, [](auto& x, auto& y) { x.swap(y); }); }
  void copyFrom(Ctx& c, DocBufs& o, size_t n) { ensure(c, n + 1); each(o, [&](auto& x, auto& y) { d2d(c, x.p, y.p, n * sizeof(*x.p)); }); }   // rows [0, n) of `o`
};

// Host state of the document. An applyChanges call works on a copy and commits it by assignment; load, reset and clone set it whole.
struct DocState {
  std::vector<std::string> actorIds;           // raw bytes, index = document actor number
  std::vector<std::pair<u32, u32>> actorRep;   // arena (offset, length) of each actor's id bytes
  std::vector<u64> clock;                      // per actor number
  u64 maxOp = 0;
  std::vector<std::array<u8, 32>> heads; std::vector<u32> headIdx;   // heads (sorted by hash) and their application indices
};

struct HostClock {
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  float ms() const { return std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};

// Timing of the last applyChanges call, and the development trace. phase(name) ends the running pipeline phase and
// starts the next one (nullptr: ends the last): a CUDA event on the main stream, a host clock mark and an NVTX range
// (nsys timelines; SURVEY.md section 5). mark(label) records a labelled host mark (amg_debug_marks). Both do nothing
// outside a call. With AMG_TRACE set (read when a call starts), the marks are printed to stderr as they happen (to see
// where a call is stuck), and load, save and the history reconstruction print theirs too, after a sync.
struct Trace {
  float ms[24] = {0};   // [0..11] CUDA-event phases, [12..23] host clock marks (ms since the call started), [23] the whole ABI call
  std::vector<std::pair<const char*, float>> marks; bool live = false;
  static bool enabled() { return getenv("AMG_TRACE") != nullptr; }
  explicit Trace(Ctx& c) : ctx(c) {}
  void begin(const char* first) { nEv = 0; record(); clk = HostClock(); for (auto& x : ms) x = 0; marks.clear(); nHost = 12; active = true; live = enabled(); nvtx(first); }
  void phase(const char* next) { if (!active) return; record(); if (nHost < 24) ms[nHost++] = clk.ms(); nvtx(next); }
  void mark(const char* label) {
    if (!active) return;
    marks.emplace_back(label, clk.ms());
    if (live) { fprintf(stderr, "amgpu mark %-28s %9.3f ms\n", label, clk.ms()); fflush(stderr); }
  }
  void end() { nvtx(nullptr); active = false; }
  // load / save / history reconstruction: host marks since `t0`, printed only with AMG_TRACE (after a sync, so they include the device work)
  void print(const char* what, const char* label, const HostClock& t0) { if (enabled()) { sync(ctx); fprintf(stderr, "amgpu %s: %-28s %9.2f ms\n", what, label, t0.ms()); } }
#ifndef AMG_EMU
  ~Trace() { if (evReady) for (auto& e : ev) cudaEventDestroy(e); }
  void collect() { cudaEventSynchronize(ev[nEv - 1]); for (int i = 0; i + 1 < nEv && i < 12; i++) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]); }   // device intervals into ms[0..11]
 private:
  cudaEvent_t ev[13]; bool evReady = false, nvtxOpen = false;   // the events are created once: 13 new timing events per call cost more than a phase
  void record() { if (!evReady) { for (auto& e : ev) cudaEventCreate(&e); evReady = true; } if (nEv < 13) cudaEventRecord(ev[nEv++], ctx.stream); }
  void nvtx(const char* name) { if (nvtxOpen) nvtxRangePop(); nvtxOpen = name != nullptr; if (name) nvtxRangePushA(name); }
#else
  void collect() {}
 private:
  void record() {} void nvtx(const char*) {}
#endif
  Ctx& ctx; HostClock clk; bool active = false; int nEv = 0, nHost = 12;
};

// Device span of the last call of each entry point kind (amg_last_*_ms): CUDA events on the main stream around the call's
// uploads, kernels and read-backs; 0 in the emulation build. start(k) zeroes k's slot and opens the span, resume(k) opens
// it without zeroing, stop() adds the span to the slot. A call that throws never reaches stop(): its slot stays 0.
enum SpanKind { SPAN_SYNC, SPAN_DECODE, SPAN_ENCODE, SPAN_HISTORY, SPAN_MERGE, SPAN_LOCAL, SPAN_GRAPH, NUM_SPANS };
struct DeviceSpans {
  float ms[NUM_SPANS] = {0};
  explicit DeviceSpans(Ctx& c) : ctx(c) {}
  void start(SpanKind k) { ms[k] = 0; resume(k); }
  void resume(SpanKind k); void stop();
#ifndef AMG_EMU
  ~DeviceSpans() { for (auto& e : ev) if (e) cudaEventDestroy(e); }
  cudaEvent_t ev[2] = {nullptr, nullptr};
#endif
  Ctx& ctx; SpanKind kind = SPAN_SYNC;
};

struct PatchOut {   // flat patch, written straight into the engine's pinned output buffer (layout: include/amgpu.h)
  u64 maxOp = 0, pendingChanges = 0; bool hasActorSeq = false; std::string actor; u64 seq = 0;
  std::vector<std::pair<u32, u64>> clock; std::vector<std::array<u8, 32>> deps; std::vector<std::string> actors;
  size_t propsOff = 0, numProps = 0, editsOff = 0, numEdits = 0, elemOff = 0, valBytesOff = 0, valBytesLen = 0, bigEnd = 0;   // byte offsets into Engine::patchBuf
  const u8* bytes = nullptr; size_t bytesLen = 0;   // final serialised patch (valid until the next call on the same engine)
};

struct HostChange { u32 off, len; };   // (arena offset, length) of the inflated change

// What the engine keeps of a document it loaded (Backend.load). loadDocument sets it whole and reset() clears it.
struct LoadedDoc {
  std::string bytes;                      // the document as loaded: what save() returns until a change is applied (new.js:2034)
  size_t numChanges = 0;                  // changes [0, numChanges) came from the document
  HostChange cols[NUM_CHANGE_COLS] = {};  // arena ranges of its change metadata columns (save() re-encodes them with later changes appended)
  bool haveHashGraph = true;              // false after a load until computeHashGraph has rebuilt the changes' bytes and hashes (new.js:1887-1912)
  size_t historyRebuilt = 0;              // changes [0, historyRebuilt) were rebuilt by computeHashGraph (getChanges DEFLATEs the large ones like encodeChange does)
  bool headIndexesUnknown = false;        // several heads and no head indexes, until computeHashGraph has matched them
};

// Pinned host mirror of the arena: grows without zero-filling; H2D copies read straight from it.
struct HostArena {
  HBuf<u8> buf; size_t len = 0;
  u8* data() { return buf.p; } const u8* data() const { return buf.p; }
  size_t size() const { return len; }
  void reserve(size_t n) { buf.ensure(n + 64); }
  void resize(size_t n) { if (n > len) buf.ensure(n + 64); len = n; }
  void append(const void* p, size_t n) { const size_t at = len; resize(len + n); memcpy(buf.p + at, p, n); }
  void assign(const HostArena& o) { resize(o.len); if (o.len) memcpy(buf.p, o.buf.p, o.len); }
};

inline std::string inflateRawBytes(const u8* p, size_t n) {
  z_stream zs; memset(&zs, 0, sizeof(zs));
  if (inflateInit2(&zs, -15) != Z_OK) throw Error(AMG_ERR_INTERNAL, "inflateInit failed");
  std::string out; out.resize(std::max<size_t>(n * 6, 1024)); zs.next_in = (Bytef*)p; zs.avail_in = (uInt)n; size_t produced = 0;
  while (true) {
    zs.next_out = (Bytef*)out.data() + produced; zs.avail_out = (uInt)(out.size() - produced);
    int rc = inflate(&zs, Z_NO_FLUSH); produced = out.size() - zs.avail_out;
    if (rc == Z_STREAM_END) break;
    if (rc != Z_OK && rc != Z_BUF_ERROR) { inflateEnd(&zs); throw Error(AMG_ERR_RANGE, "invalid deflate data"); }
    if (zs.avail_out == 0) out.resize(out.size() * 2); else if (zs.avail_in == 0) { inflateEnd(&zs); throw Error(AMG_ERR_RANGE, "unexpected end of deflate data"); }
  }
  inflateEnd(&zs); out.resize(produced); return out;
}
inline std::string deflateRawBytes(const u8* p, size_t n) {   // zlib level 6, as pako.deflateRaw
  z_stream zs; memset(&zs, 0, sizeof(zs));
  if (deflateInit2(&zs, 6, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) throw Error(AMG_ERR_INTERNAL, "deflateInit failed");
  std::string comp; comp.resize(deflateBound(&zs, (uLong)n));
  zs.next_in = (Bytef*)p; zs.avail_in = (uInt)n; zs.next_out = (Bytef*)comp.data(); zs.avail_out = (uInt)comp.size();
  const int rc = ::deflate(&zs, Z_FINISH); comp.resize(zs.total_out); deflateEnd(&zs);
  if (rc != Z_STREAM_END) throw Error(AMG_ERR_INTERNAL, "deflate failed");
  return comp;
}
inline std::string hex_of(const u8* p, size_t n) { static const char* d = "0123456789abcdef"; std::string s; for (size_t i = 0; i < n; i++) { s.push_back(d[p[i] >> 4]); s.push_back(d[p[i] & 15]); } return s; }

class Engine {
 public:
  Ctx ctx;
  // ---- persistent device state
  DBuf<u8> arena; size_t arenaLen = 0; HostArena hostArena;   // pinned host mirror (values / keys / changes are read from it)
  DBuf<u8> hashes; size_t numApplied = 0;
  DocBufs doc; size_t numRows = 0; DBuf<u32> succOff; DBuf<u64> succ; size_t numSucc = 0;
  DBuf<ActorSlot> actorSlots; size_t actorCap = 0;
  DBuf<u32> actorRank;
  // application index of each actor's last applied change (by document actor number; set by commit, load and clone).
  // commit() swaps in lastChangeNext, which the sequence check of the call filled.
  DBuf<u32> lastChange, lastChangeNext;
  // ---- persistent host state
  DocState st;
  std::vector<HostChange> changes;     // applied, in application order
  struct OrigRange { u32 idx; HostChange range; };
  std::vector<OrigRange> deflatedOriginal;        // (applied change index, arena range of the original DEFLATEd bytes), ascending index
  const HostChange* originalOf(u32 idx) const {
    auto it = std::lower_bound(deflatedOriginal.begin(), deflatedOriginal.end(), idx, [](const OrigRange& a, u32 v) { return a.idx < v; });
    return it != deflatedOriginal.end() && it->idx == idx ? &it->range : nullptr;
  }
  std::vector<HostChange> queue, queueOriginal;   // not yet causally ready (+ original range, len 0 = not deflated)
  std::vector<u32> deflateOnExport;   // ascending applied indexes of changes a merge applied in plain form where getChangesAdded hands them over DEFLATEd
  // getChanges & co hand change idx out DEFLATEd, as encodeChange returns a change of 256 bytes or more (columnar.js:738):
  // a change rebuilt by computeHashGraph, or one a merge applied in plain form. A change that arrived DEFLATEd goes out as
  // its original bytes instead (originalOf).
  bool exportsDeflated(u32 idx) const {
    if (changes[idx].len < 256 || originalOf(idx)) return false;
    return idx < loaded.historyRebuilt || std::binary_search(deflateOnExport.begin(), deflateOnExport.end(), idx);
  }
  Trace trace{ctx};
  HBuf<u8> patchBuf;   // pinned: patch records are copied device -> host directly into their final place
  DeviceSpans spans{ctx};   // sync, decode, encode, history, merge, local-change and graph-query calls
  // ---- scratch (grow-only)
  DBuf<u32> chOff, chLen, nOps, nPreds, nDeps, nActors, colOff, colLen, depBase, depIdx, primary, pass, flagWord, appRank, opBase, predBase, timeBase, amapBase, amap, authorSlot, newSlots;
  DBuf<u8> applied; DBuf<ChangeHot> hot; DBuf<ChangeMeta> meta /* save(): full headers */; DBuf<u64> errWord; DBuf<u32> hashTable;
  DBuf<u32> inflCap, inflCapOff, inflOvf; DBuf<u8> inflScratch; DBuf<u64> inflTotal;
  u64 inflateSpeculate(InflateArgs& ia);   // first inflate pass + inflOff; returns the 64-bit total of the inflated sizes
  DBuf<u32> rawBase, rawPredBase, decErr, decDirect; DBuf<u64> decCursor; size_t lastDeflCount = 0, lastDeflStart = 0;
  u32* decTotalsPtr() { return reinterpret_cast<u32*>(decCursor.p + 2); }
  DBuf<u32> patchByteLen, patchByteOff; DBuf<u8> patchBytesD;   // key / value bytes shipped inside the patch   // fused decode (decode.cuh k_decode_tiles)
  DBuf<u32> r_objActor, r_objCtr, r_keyActor, r_keyCtr, r_keyStrOff, r_keyStrLen, r_insert, r_action, r_valLen, r_valOff, r_predNum, r_predOff, r_predActor, r_predCtr;
  DBuf<u64> o_id, o_obj, o_key, o_predId; DBuf<u32> o_keyStrOff, o_keyStrLen, o_flags, o_valLen, o_valOff, o_predOff, o_predNum, o_change, o_time;
  DBuf<u32> isRow, rowSlot, rowOfOp; DocBufs work, sorted;
  DBuf<u64> idKeys; DBuf<u32> idVals; DBuf<u32> objRow, elemRow, parentRow, keySlot, repList, repCount, listPos, perm, pos;
  DBuf<KeySlot> keySlots; DBuf<u64> sortKeys; DBuf<u32> sortVals; SortTemp sortTmp; ScanTemp scanTmp;
  ParColumnDecoder parCols{ctx, scanTmp}; size_t parDocMinRows = 4096;   // documents with at least this many rows decode their columns in parallel (doccols.cuh); AMG_PAR_DOC_MIN overrides
  DBuf<u32> eNext, eRank, insItems, itemIdx, objSlot; DBuf<u64> ePacked, ePacked2;
  DBuf<u64> pairKey, pairSucc, newSucc; DBuf<u32> pairIdx, pairPos, pairTime, succCnt, newSuccCnt, newSuccOff, firstNewSucc;
  DBuf<u32> elemPos, keyRankAt, objPos, head, headScan, groupOf, groupRows, groupVisible, groupFirst, groupTouched, groupLinked, objTouchedAt, linkDone, emit, marker, slot;
  DBuf<u32> isObjHead, objIdx, objStart, elemVis, elemVisScan, rowEmit, firstVis, state, nItems, itemBase, qIndex, zero, wzero, zscan, wscan, editObjKey;
  DBuf<DomItem> items, items2; DBuf<PropRec> propOut; DBuf<EditRec> editOut, editOut2; DBuf<u64> editElem, editElem2;
  std::unique_ptr<ColumnEncoder> encoder; DBuf<long long> saveVals; DBuf<u32> saveStrOff, saveStrLen; DBuf<u64> counterTotal; DBuf<int> domW, domW2; DBuf<u32> elemMinT, editRowPos, editRowPos2, editObjKey2, rowClass, firstBare, counterOwner, newSuccTime, counterLast, runHeadFlag, runScan, runStart, elemFollower, domTw, domTw2, oldVisScan, inflLen, inflOff, groupHasChild, gCount, gElem, gT1, gQOrd, gBase, nQ, elemHasRecs, listLinkTime, editElemPos, editElemPos2, editKind, editPred, editDead, editMerge, editMulti, editLive;
  DBuf<u32> seqSlot, actorCnt, actorBaseD, clockD, changeActor, editTime; DBuf<u8> hashTmp; DBuf<u32> headsPack, headsOut;
  DBuf<u32> finalTime, gFailed, memberFinal, opAt, runHead, opGroupHead; DBuf<u64> gBound; DBuf<HostChange> chPairs; DBuf<u32> largeFlag, largeSlot, largeList; size_t lastNumLarge = 0; DBuf<u64> zwScan; DBuf<u32> deflList, patchTriples;

  explicit Engine(int device) {
    ctx.device = device;
#ifndef AMG_EMU
    int count = 0; cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) throw Error(AMG_ERR_CUDA, "amgpu: no CUDA device available (this library has no CPU fallback)");
    CUDA_CHECK(cudaSetDevice(device));
    cudaDeviceProp prop; CUDA_CHECK(cudaGetDeviceProperties(&prop, device)); ctx.numSMs = prop.multiProcessorCount;
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx.stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx.side, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx.copy, cudaStreamNonBlocking));
    ctx.peekCap = 1u << 20; CUDA_CHECK(cudaMallocHost((void**)&ctx.peekBuf, ctx.peekCap + 64));
    ctx.peekFlag = reinterpret_cast<volatile unsigned long long*>(ctx.peekBuf + ctx.peekCap); *ctx.peekFlag = 0;
    CUDA_CHECK(cudaEventCreateWithFlags(&ctx.evUp, cudaEventDisableTiming)); CUDA_CHECK(cudaEventCreateWithFlags(&ctx.evMirror, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&ctx.evFork, cudaEventDisableTiming)); CUDA_CHECK(cudaEventCreateWithFlags(&ctx.evJoin, cudaEventDisableTiming));
    ShaConsts k; memcpy(k.k, SHA_K, sizeof(SHA_K)); CUDA_CHECK(cudaMemcpyToSymbol(c_sha, &k, sizeof(k)));
#endif
    errWord.ensure(ctx, 4); flagWord.ensure(ctx, 16);
    actorCap = 64; actorSlots.ensure(ctx, actorCap); rebuildActorTable();
    succOff.ensure(ctx, 1); dev_memset(ctx, succOff.p, 0, 4);
  }
  ~Engine() {
#ifndef AMG_EMU
    if (ctx.stream) cudaStreamDestroy(ctx.stream);
    mirror_wait(ctx);
    if (ctx.side) cudaStreamDestroy(ctx.side);
    if (ctx.copy) cudaStreamDestroy(ctx.copy);
    if (ctx.peekBuf) cudaFreeHost(ctx.peekBuf);
    if (last_peek_ctx() == &ctx) last_peek_ctx() = nullptr;
    if (ctx.evUp) cudaEventDestroy(ctx.evUp);
    if (ctx.evMirror) cudaEventDestroy(ctx.evMirror);
    if (ctx.evFork) cudaEventDestroy(ctx.evFork);
    if (ctx.evJoin) cudaEventDestroy(ctx.evJoin);
#endif
  }

  // (re)builds the device actor table from the host's actor list (after growth, rollback or commit)
  void rebuildActorTable() {
    std::vector<ActorSlot> t(actorCap); for (auto& s : t) { s.hash = 0; s.first = ~0ULL; s.actorNum = EMPTY32; s.repOff = 0; s.repLen = 0; s.pad = 0; }
    for (size_t a = 0; a < st.actorIds.size(); a++) {
      const u64 h = fnv1a64((const u8*)st.actorIds[a].data(), (u32)st.actorIds[a].size()); u64 s = mix64(h) & (actorCap - 1);
      while (t[s].hash != 0) s = (s + 1) & (actorCap - 1);
      t[s].hash = h; t[s].first = 0; t[s].actorNum = (u32)a; t[s].repOff = st.actorRep[a].first; t[s].repLen = st.actorRep[a].second;
    }
    h2d(ctx, actorSlots.p, t.data(), actorCap * sizeof(ActorSlot)); sync(ctx);
  }

  // ---------------------------------------------------------------- error plumbing
  // Every small device -> host read also brings the error word along (same sync); a later error check is free when no
  // kernel was launched in between.
  u64 errSnapshot = 0; uint64_t errSnapLaunches = ~0ull;
  u64* pinnedWords(size_t n) { hostWord.ensure(n + 1); return hostWord.p; }
  void readWords(std::initializer_list<std::pair<const void*, size_t>> srcs, void* const* dsts) {   // one sync for all of them + the error word
    u64* w = pinnedWords(srcs.size() + 1); size_t k = 0;
    const void* from[9]; size_t sizes[9]; void* to[9];
    if (srcs.size() > 8) throw Error(AMG_ERR_INTERNAL, "readWords: too many words");
    for (auto& s : srcs) { w[k] = 0; from[k] = s.first; sizes[k] = s.second; to[k] = &w[k]; k++; }
    from[k] = errWord.p; sizes[k] = 8; to[k] = &w[k];
#ifndef AMG_EMU
    ctx.peekFlagArmed = false;
#endif
    if (k + 1 <= 8) d2h_words(ctx, (int)k + 1, from, sizes, to); else for (size_t i = 0; i <= k; i++) d2h(ctx, to[i], from[i], sizes[i]);
    const uint64_t launchesNow = ctx.launches;
    sync(ctx, true);   // the words' kernel is the last thing on the stream: wait on its completion flag
    k = 0; for (auto& s : srcs) { memcpy(dsts[k], &w[k], s.second); k++; }
    errSnapshot = w[k]; errSnapLaunches = launchesNow;
  }
  u64 fetchErr() { if (errSnapLaunches != ctx.launches) { void* none[1] = {nullptr}; readWords({}, none); } return errSnapshot; }
  void clearErr() { dev_memset(ctx, errWord.p, 0, 16); errSnapLaunches = ~0ull; }   // the next check reads the word again
  static std::string opIdText(u64 id, const std::vector<std::string>& actors) {
    const u32 a = id_actor(id);
    return std::to_string(id_ctr(id)) + "@" + (a < actors.size() ? hex_of((const u8*)actors[a].data(), actors[a].size()) : std::string("?"));
  }
  [[noreturn]] static void throwKernelError(u64 w) {
    const u32 code = (u32)(w & 0xff);
    switch (code) {
      case KE_MAGIC: throw Error(AMG_ERR_RANGE, "Data does not begin with magic bytes 85 6f 4a 83");
      case KE_CHECKSUM: throw Error(AMG_ERR_RANGE, "checksum does not match data");
      case KE_TRAILING: throw Error(AMG_ERR_RANGE, "Encoded change has trailing data");
      case KE_CHUNK_TYPE: throw Error(AMG_ERR_RANGE, "Unexpected chunk type");
      case KE_DEFLATE: throw Error(AMG_ERR_RANGE, "invalid deflate data");
      case KE_HIST_RANGE: throw Error(AMG_ERR_RANGE, "Operation ID outside of allowed range");        // columnar.js:925
      case KE_HIST_OPID: throw Error(AMG_ERR_RANGE, "Expected opId does not match the operation found");   // columnar.js:936
      case KE_HIST_DEP: throw Error(AMG_ERR_RANGE, "No hash for dependency index");                      // columnar.js:952
      case KE_TRUNCATED: throw Error(AMG_ERR_RANGE, "buffer ended with incomplete number");
      case KE_SUBARRAY: throw Error(AMG_ERR_RANGE, "subarray exceeds buffer size");
      case KE_NUM_RANGE: throw Error(AMG_ERR_RANGE, "number out of range");
      case KE_COL_ORDER: throw Error(AMG_ERR_RANGE, "Columns must be in ascending order");
      case KE_COL_DEFLATE: throw Error(AMG_ERR_RANGE, "change must not contain deflated columns");
      case KE_RLE_REP1: throw Error(AMG_ERR_RANGE, "Repetition count of 1 is not allowed, use a literal instead");
      case KE_RLE_SUCC_REP: throw Error(AMG_ERR_RANGE, "Successive repetitions with the same value are not allowed");
      case KE_RLE_SUCC_LIT: throw Error(AMG_ERR_RANGE, "Successive literals are not allowed");
      case KE_RLE_SUCC_NULL: throw Error(AMG_ERR_RANGE, "Successive null runs are not allowed");
      case KE_RLE_ZERO_NULL: throw Error(AMG_ERR_RANGE, "Zero-length null runs are not allowed");
      case KE_RLE_LIT_REP: throw Error(AMG_ERR_RANGE, "Repetition of values is not allowed in literal");
      case KE_BOOL_ZERO: throw Error(AMG_ERR_RANGE, "Zero-length runs are not allowed");
      case KE_OBJ_MISMATCH: throw Error(AMG_ERR_RANGE, "Mismatched object reference");
      case KE_KEY_MISMATCH: throw Error(AMG_ERR_RANGE, "Mismatched operation key");
      case KE_ACTOR_INDEX: throw Error(AMG_ERR_RANGE, "actor index out of range");
      case KE_TOO_LARGE: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: value exceeds the engine's 32-bit counter / 4 GiB arena limits");
      case KE_UNKNOWN_ACTOR: throw Error(AMG_ERR_RANGE, "actorId is not known to document");
      case KE_PRED_MISSING: throw Error(AMG_ERR_RANGE, "no matching operation for pred");
      case KE_REF_ELEM: throw Error(AMG_ERR_RANGE, "Reference element not found");
      case KE_LIST_ELEM: throw Error(AMG_ERR_RANGE, "could not find list element with ID");
      case KE_DUP_OPID: throw Error(AMG_ERR_RANGE, "duplicate operation ID");
      case KE_LAMPORT: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: insert with an opId not greater than its reference element (Lamport order violated)");
      case KE_HASH_COLLISION: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: 64-bit string hash collision");
      case KE_GROUP_COLUMN: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: a GROUP_CARD column of an unknown version in the group of known columns (the reference would read those as arrays)");
      case KE_UNSUPPORTED_OP: throw Error(AMG_ERR_UNSUPPORTED, "amgpu: operation pattern outside the incremental-patch subset (see DESIGN.md)");
      default: throw Error(AMG_ERR_INTERNAL, "amgpu: kernel error " + std::to_string(code));
    }
  }
  void checkErr() { u64 w = fetchErr(); if (w) throwKernelError(w); }

  // ---------------------------------------------------------------- helpers
  DBuf<u64> gateBest;   // causal gate with several copies of a waiting change: best (pass, position) per hash
  bool domLocalReady = false;   // k_dom_local's dynamic shared memory size has been raised on this device
  std::vector<HostChange> batchStore;   // applyChanges: (offset, length) of the batch entries
  HBuf<HostChange> pairStage;           // the same table in pinned memory: uploaded by DMA
  HBuf<u32> pinnedScratch; HBuf<u64> hostWord;   // pinned landing slots for the small device -> host reads that size the next stage
  u32 readU32(const u32* dptr) { u32 v = 0; void* d[1] = {&v}; readWords({{dptr, 4}}, d); return v; }
  void readU32x2(const u32* a, const u32* b, u32* va, u32* vb) { void* d[2] = {va, vb}; readWords({{a, 4}, {b, 4}}, d); }
  void fill32(u32* p, u32 v, size_t n) { foreach(ctx, n, FillU32Kernel{p, v}); }
  u64 hashTableOf(const u8* hs, size_t count);   // hashTable over hashes [0, count); returns its slot mask
  u32 parseChangeHeaders(const u8* ar, const HostChange* pairs, size_t K);   // then resolveChangeDeps: dependency indexes from change headers
  u64 resolveChangeDeps(const u8* ar, const u8* hs, size_t C, size_t K, size_t base, u32 totalDeps);
  // sort `perm` (row ids) by successive 64-bit fields produced by keyFn(field) ; stable LSD over fields
  void sortPairs(DBuf<u64>& keys, DBuf<u32>& vals, size_t n, int bits) { radix_sort_pairs(ctx, sortTmp, keys, vals, n, 0, bits); }

  // reference columnar.js:813-823 (pako.inflateRaw -> zlib raw inflate); magic + checksum are kept
  static std::string inflateChange(const u8* buf, size_t len) {
    ByteReader r(buf, 9, (u32)len); const u64 clen = r.uleb();
    if (r.err || r.pos + clen > len) throw Error(AMG_ERR_RANGE, "buffer ended with incomplete number");
    const std::string body = inflateRawBytes(buf + r.pos, clen);
    // header: magic + checksum (8 bytes), chunk type 1, LEB128 length, then the inflated body
    std::string out((const char*)buf, 8); out.push_back(1); put_uleb(out, body.size());
    return out + body;
  }

  // ---------------------------------------------------------------- applyChanges
  // What one call's phases hand to each other (engine_impl.cuh). Device scratch stays in the engine: grow-only, reused.
  struct ApplyCall {
    const u8* const* bufs; const size_t* lens; size_t n; const u8* blob; const u64* offsets; bool isLocal, wantPatch;   // pointer array or packed blob
    // merge: per new entry, 1 = goes out DEFLATEd once applied (Engine::deflateOnExport). A merge batch is causally complete
    // over the document (every dependency is applied or in the batch), so no marked entry is left waiting in the queue.
    const u8* exportMarks = nullptr;
    enum { SRC_PINNED, SRC_DEVICE, SRC_PAGEABLE } srcKind = SRC_PAGEABLE; bool offsetsByDma = false, copiesFirst = false;
    size_t total = 0, arenaLen0 = 0, cur = 0, Bq = 0, B = 0;   // batch: n new changes, then Bq queued ones; bytes arena[arenaLen0, cur)
    size_t queueBytes = 0;   // bytes of the Bq queued entries: they lie before arenaLen0, outside [arenaLen0, cur)
    struct Piece { size_t byteEnd, changeEnd, mark; }; std::vector<Piece> pieces;
    HostChange* pairs = nullptr; u8* hashOut = nullptr; DecodeTilesArgs dargs{};   // pairs: pinned (offset, length) table of the batch
    // DEFLATEd changes: originals of queue entries (batchOriginal, dense) and of the ones inflated now (inflOrig, parallel to deflIdx)
    std::vector<HostChange> batchOriginal, inflOrig; std::vector<u32> deflIdx; size_t inflNd = 0, inflExtraStart = 0, inflExtra = 0; bool inflPending = false;
    void finishInflate(Engine& e); HostChange originalOf(size_t b) const;
    u32 decTot[4] = {0, 0, 0, 0};   // decode totals: ops, preds, overflow, flags (1: large changes, 2: unknown columns)
    size_t G = 0, numNew = 0; bool inOrder = true; u32 D = 0;   // gate: G = applied before + batch; D dependency entries
    std::vector<u8> appliedH; std::vector<u32> primaryH, appRankH; std::vector<HostChange> newQueue, newQueueOriginal;   // host copies: only when an entry waits or the order differs
    DocState now;   // the document's host state as this call leaves it
    size_t M = 0, P = 0, N = 0, numPairs = 0; OpRows ops{}; IdTable idt{nullptr, nullptr, 0}; Ord ord{}; DocRows w{};   // w: rows before the sort
    std::vector<std::pair<u64, UnknownRow>> unknownRows; std::set<u32> unknownIds;
    std::thread fill;   // fills the host's list of the batch entries; needBatch() joins it before the list is first read
    void needBatch() { if (fill.joinable()) fill.join(); }
    ~ApplyCall() { needBatch(); }
  };
  void applyChanges(const u8* const* bufs, const size_t* lens, size_t n, const u8* blob, const u64* offsets, bool isLocal, bool wantPatch, PatchOut& out,
                    const u8* exportMarks = nullptr);
  void applyChangesOnce(ApplyCall& a, PatchOut& out);   // the phases, in order:
  void stageBatch(ApplyCall& a), inflateBatch(ApplyCall& a), runGate(ApplyCall& a), internActors(ApplyCall& a), checkSequence(ApplyCall& a), finalizeOps(ApplyCall& a),
       orderOpSet(ApplyCall& a), computeHeads(ApplyCall& a), commit(ApplyCall& a);
  void queueCopy(ApplyCall& a, ApplyCall::Piece& pc, size_t byte0, size_t ch0); void fillPairs(ApplyCall& a);
  // error messages of the rare paths
  [[noreturn]] void throwActorError(u64 ew, const std::vector<std::string>& actors); [[noreturn]] void throwSequenceError(ApplyCall& a);
  [[noreturn]] void throwOpError(u64 ew, const std::vector<std::string>& actors); [[noreturn]] void throwPatchValueError(u64 ew, size_t numProps);
  void getPatch(PatchOut& out);
  struct PatchInputs {   // everything buildPatch reads: the rows in document order, their succ CSR and counts; incremental: the batch and the op-set tables
    DocRows d; size_t N; bool wholeDoc; const u32* succOff; const u64* succ; const u32* succCnt; Ord ord;
    const OpRows* ops = nullptr; size_t numOps = 0; const IdTable* idt = nullptr; const u32 *rowOfOp = nullptr, *pos = nullptr;
    const u32 *newSuccCnt = nullptr, *firstNewSucc = nullptr, *newSuccTime = nullptr, *objPos = nullptr, *pass = nullptr; DocRows unsorted{};   // rows before the sort
  };
  void buildPatch(const PatchInputs& in, PatchOut& out);
  void fillPatchHeader(PatchOut& out);
  void finishPatch(PatchOut& out);
  void reset();
  DBuf<u64> excl64, offsDev;
  void benchDecode(int iters, float* msSha, float* msParse, float* msDec, u64* algoBytes);
  UnknownStore unknownCols;   // values of columns with ids this version does not know, per op (unknowncols.hpp)
  void collectUnknownColumns(size_t B, std::vector<std::pair<u64, UnknownRow>>& out, std::set<u32>& ids);
  void appendUnknownDocColumns(std::vector<std::pair<u32, std::string>>& cols);   // save(): their document columns
  RawRows rawRows();
  void decodeHugeChanges(const RawRows& raw, size_t numLarge); DBuf<u32> hugeDone;
  void runDecodeTiles(const u8* arenaP, size_t B, size_t batchBytes, const u32* deflListP = nullptr, size_t numDefl = 0, size_t deflStart = 0);
  DecodeTilesArgs decodeArgs(const u8* arenaP, size_t B, size_t batchBytes);
  // Host mirror of the arena, filled on demand: hostArena holds arena[0, hostArena.size()); whatever is missing is fetched
  // from the device when a reader (getChanges, amg_arena, clone ...) asks for it.
  void ensureHostMirror() {
    if (hostArena.size() >= arenaLen) return;
    const size_t from = hostArena.size(); hostArena.resize(arenaLen);
    d2h(ctx, hostArena.data() + from, arena.p + from, arenaLen - from); sync(ctx);
  }   // sizes the raw row tables and launches the fused decode
  bool decodeOverflowed(const u32 totals[4]);
  int debugDecodeColumn(const u8* bytes, size_t len, int kind, size_t n, bool parallel, long long* out);
  void decodeRaw(const u8* blob, const u64* offsets, size_t n, u8* hashesOut, u32* nOpsOut, u32** rowsOut, size_t* totalOps, size_t* totalPreds);
  size_t lastB = 0, lastM = 0, lastP = 0, lastBytes = 0;
  size_t decWantRows = 0, decWantPreds = 0, decRowCap = 0, decPredCap = 0;

  // ---------------------------------------------------------------- load, save, history: what one call's phases hand to each other
  LoadedDoc loaded;
  void decodeLoadedCol(int k, size_t count, long long* out, u32* strOff, u32* strLen);   // change metadata column k of the loaded document
  struct LoadCall {
    const u8* buf; size_t len; ByteReader r; HostClock t0;
    struct ColInfo { u32 id; u64 len; std::string data; }; std::vector<ColInfo> changeCols, opCols;
    std::vector<std::pair<ColInfo*, const u8*>> deflated;   // columns still DEFLATEd, and where their bytes are
    std::vector<std::string> actors; std::vector<std::array<u8, 32>> heads; std::vector<u32> headIdx;
    std::vector<std::pair<u32, u32>> reps; DocCols dc{}; size_t arenaLen = 0;   // staged in the arena
    std::vector<u64> clock; std::vector<u32> lastChange; LoadedDoc doc;   // doc: what the engine keeps once the load has succeeded
    size_t N = 0, S = 0; u32 serialMask = ALL_DOC_COLS; bool counted = false; RawRows raw{}; u64 maxOp = 0;   // rows, succ entries
    LoadCall(const u8* b, size_t n) : buf(b), len(n), r(b, 8, (u32)n) {}
  };
  void loadDocument(const u8* buf, size_t len);   // the phases, in order:
  void readContainer(LoadCall& l), inflateColumns(LoadCall& l), stageColumns(LoadCall& l), loadClock(LoadCall& l), countRows(LoadCall& l),
       decodeDocColumns(LoadCall& l), finalizeRows(LoadCall& l), readUnknownOpColumns(LoadCall& l), commitLoad(LoadCall& l);
  void ensureLoadRows(size_t n);
  struct SaveCall {
    size_t C, N, S, L, K;   // changes, rows, succ entries, loaded changes; the K = C - L later ones have their bytes in the arena
    struct Col { u32 id; size_t off, len; }; std::vector<Col> changeCols, opCols;   // ranges of the encoder's output
    HostClock t0;
  };
  void saveDocument(std::string& result);   // the phases, in order:
  void saveChangeColumns(SaveCall& s), saveOpColumns(SaveCall& s); void packDocument(SaveCall& s, std::string& result);
  // Change metadata of every applied change (save() and historyPatches): the first L from the loaded document's columns, the
  // K = C - L later ones from their headers in the arena (ParseKernel, their dependency hashes resolved to change indexes).
  // parseChangeMeta fills the engine's meta / depIdx scratch; changeMetaColumn then writes column `col` (CHANGE_COLS
  // index) for all C changes, or for the loadedDeps + laterDeps dependency indexes.
  struct ChangeMetaCall { size_t C, L, K; u32 loadedDeps = 0, laterDeps = 0; };
  void parseChangeMeta(ChangeMetaCall& m);
  void changeMetaColumn(const ChangeMetaCall& m, int col, long long* out, u32* strOff, u32* strLen);
  // computeHashGraph's tables live as long as the call (they go back to the pool when it ends)
  struct HistoryCall {
    size_t L, N, S, A; DocRows d; HostClock t0;
    DBuf<long long> cActor, cSeq, cMaxOp, cTime, cDepsNum, cExtra, depIdxV, scratchV; DBuf<u32> msgOff, msgLen, extraOff, extraLen, tmpOff, tmpLen, depsNum32, depBase, depIdx; size_t D = 0;
    DBuf<u32> rankD, actorOfRank, repOff, repLen; int ctrBits = 0, idBits = 0;
    DBuf<u64> idSorted, predKey, succKey, keyA, keyB, groupId, opId; size_t G = 0, numDel = 0, M = 0;
    DBuf<u32> idRows, pairRow, valA, pairRowSorted, head, groupIdx, groupStart, groupRow, isDel, delSlot, opSrc, opPredStart, opPredNum, opOrder, opChange, predNumSorted, opPredBase;
    DBuf<u64> opKey, chKey; DBuf<u32> changeOrder, actorStart, chOpStart, chNOps; size_t P = 0;
    DBuf<u32> slotCnt, slotBase, uniq, uniqSlot, otherStart, slotVal; DBuf<u64> slotKey, other; size_t Q = 0, U = 0;
    DBuf<u32> objA, keyAi, predA, outLen, outOff, depsAt, bodyAt, chOffD; DBuf<long long> keyDelta, predDelta; u64 T = 0;
    DBuf<u32> listD; DBuf<u8> newHashes; std::vector<u8> isDep;
    HistOpView view() { return HistOpView{d, opId.p, opSrc.p, opPredStart.p, opPredNum.p, opOrder.p, pairRowSorted.p, (u32)N}; }
  };
  void computeHashGraph();   // change history of a loaded document (history.cuh), once (later calls return at once); the sections, in order:
  void histChangeColumns(HistoryCall& h), histActorOrder(HistoryCall& h), histPredsAndDeletions(HistoryCall& h), histOpsToChanges(HistoryCall& h),
       histActorTables(HistoryCall& h), histEncode(HistoryCall& h), histHashes(HistoryCall& h), histCheckHeads(HistoryCall& h), histCommit(HistoryCall& h);

  // ---------------------------------------------------------------- sync protocol (sync.cuh, engine_impl.cuh)
  // Candidates are change indexes idx[0, count); idx == nullptr: every applied change, in application order. The change
  // hashes must be known (computeHashGraph has run on a loaded document).
  struct BloomSpec { u32 numEntries, numProbes; const u8* bits; size_t bitsLen; };   // a peer's parsed filter (sync.js:38-76)
  void syncBloom(const u32* idx, size_t count, std::string& out);   // BloomFilter(hashes).bytes
  void syncChangesToSend(const u32* idx, size_t count, const std::vector<BloomSpec>& filters, std::vector<u8>& send);   // send[i]: Bloom-negative or depends on one
  void gatherHashes(const std::vector<u32>& idx, std::string& out);   // 32 bytes per change
  DBuf<u32> syncIdx, syncBits; DBuf<u8> syncFilterBits, syncNeg, syncHashOut; DBuf<BloomRef> syncFilters;

  // ---------------------------------------------------------------- decodeChange / decodeChanges (changes.cuh)
  // n change containers into one flat change table (layout: include/amgpu.h). Source: the caller's blob (staged into scratch,
  // DEFLATEd changes inflated on the device behind it) or, with history, every applied change read in place from the arena.
  // The document is not touched. On error, decodeFailed names the change.
  struct DecodeCall {
    size_t n = 0; const u8* ar = nullptr; bool history = false;
    u32 tot[4] = {0, 0, 0, 0};   // ops, preds, actor table entries, bytes
    size_t changesOff = 0, opsOff = 0, predsOff = 0, actorsOff = 0, bytesOff = 0, size = 0;   // sections of the table
  };
  void decodeChanges(const u8* blob, const u64* offsets, size_t n, bool history, std::string& out);
  void stageDecodeInput(DecodeCall& d, const u8* blob, const u64* offsets), inflateDecodeInput(DecodeCall& d), decodeTable(DecodeCall& d, std::string& out);
  [[noreturn]] void throwDecodeError(DecodeCall& d, const u64* words);
  std::pair<size_t, int> firstFailingChange(const u64* words, int numPhases, int opPhase, const u32* opBaseDev, size_t n);
  size_t decodeFailed = 0;   // failing change of the last call
  DBuf<u8> dcArena, dcHash, dcOut; DBuf<u32> dcOff, dcLen, dcCLen, dcOps, dcPreds, dcActors, dcBytes, dcOpBase, dcPredBase, dcActorBase, dcByteBase, dcColOff, dcColLen, dcRows, dcChld;
  DBuf<ChangeMeta> dcMeta; DBuf<u64> dcErr, dcTotals; DBuf<u32> dcDefl;

  // ---------------------------------------------------------------- encodeChange over a change table (encchg.cuh)
  // The n changes of a change table (layout: include/amgpu.h) into plain binary changes and their hashes. The table is
  // staged like decodeChanges' input; the document is not touched. On error, encodeFailed names the change. Its tables live
  // as long as the call.
  struct EncodeCall {
    size_t n = 0; u64 len = 0; u64 hdr[CHG_HDR_WORDS] = {}; EncTable T{};
    size_t M = 0, P = 0, E = 0, Q = 0, U = 0; u32 maxActorLen = 0; u64 total = 0;   // ops, preds, actor entries, actor slots, (change, actor) pairs; output bytes
    DBuf<u64> err, totals; DBuf<u32> nOps, nPreds, nActors, opBase, predBase, actorBase, slotCnt, slotBase;
    DBuf<u32> entOff, entLen, entRank, rep, head, headScan, sortVals, uniq, uniqSlot, otherStart; DBuf<u64> sortKeys, slotKeys, other;
    DBuf<u32> objA, keyA, chA, predA, colLen, outLen; DBuf<long long> keyDelta, chDelta, predDelta; DBuf<u64> predKey, outOff, dataAt, depsAt, bodyAt;
    DBuf<u8> out, hashes;
  };
  // out: the changes back to back, offs: n + 1 offsets into it, hashes: n x 32 bytes
  void encodeChanges(const u8* table, size_t len, std::string& out, std::vector<u64>& offs, std::string& hashesOut);   // the phases, in order:
  void stageEncodeInput(EncodeCall& e, const u8* table), validateTable(EncodeCall& e), encodeActorTables(EncodeCall& e), encodePrep(EncodeCall& e),
       encodeColumns(EncodeCall& e), encodeHashes(EncodeCall& e);
  void copyEncodeOutput(EncodeCall& e, std::string& out, std::vector<u64>& offs, std::string& hashesOut);
  [[noreturn]] void throwEncodeError(EncodeCall& e, const u64* words);
  size_t encodeFailed = 0;   // failing change of the last call

  // ---------------------------------------------------------------- getHistory snapshots (snapshot.cuh)
  // The whole-document patch of the first k applied changes (getAllChanges order) for every k of a list: the op table
  // filtered to the prefix's rows and succ entries, then buildPatch as getPatch runs it. The per-change tables are built
  // once per call and shared by its prefix lengths; the document is not touched.
  struct HistoryPatchCall {
    size_t C = 0, A = 0, N = 0, S = 0, D = 0;   // applied changes, actors, rows, succ entries, dependency edges
    ChangeMetaCall m{};
    DBuf<long long> cActor, cSeq, cMaxOp, cDepsNum, depIdxV; DBuf<u32> strOff, strLen, depsNum32, depBase, depIdx;
    DBuf<u64> chKey; DBuf<u32> changeOrder, actorStart, rowChange, succChange, firstDep;
    DBuf<u32> keep, rowPos, cnt, cntPos, headFlag, headPos, headIdx; DBuf<u64> clock; DBuf<u8> headHashes;   // per prefix length
  };
  void historyPatches(const u64* prefixLens, size_t n, std::vector<std::string>& out);   // the phases, in order:
  void snapChangeMeta(HistoryPatchCall& h), snapActorOrder(HistoryPatchCall& h), snapChangeIndexes(HistoryPatchCall& h);
  size_t snapFilter(HistoryPatchCall& h, size_t k);   // per prefix length: the prefix document into snapDoc (returns its rows)
  void snapHeader(HistoryPatchCall& h, size_t k, PatchOut& out);
  DocBufs snapDoc; DBuf<u32> snapSuccOff, snapSuccCnt; DBuf<u64> snapSucc;   // the prefix document (grow-only; never the document's own)

  // ---------------------------------------------------------------- merge (merge.cuh)
  // The applied changes of `src` this document lacks, as indexes into src.changes, in the order getChangesAdded returns
  // them (new.js:1979-1997). Runs on this engine's stream and scratch; src is only read (its history is rebuilt first when
  // it was loaded, as getChangesAdded does). Both documents must be on the same device (AMG_ERR_UNSUPPORTED otherwise).
  void changesAddedFrom(Engine& src, std::vector<u32>& order);
  // Automerge.merge (src/automerge.js:61-67): those changes, gathered from src's arena into one device blob, through applyChanges
  void mergeFrom(Engine& src, bool wantPatch, PatchOut& out);
  DBuf<u32> mergeAbsent, mergeSlot, mergeList, mergeHeadIdx; DBuf<u8> mergeHeads, mergeBlob; DBuf<MergeRange> mergeRanges;

  // ---------------------------------------------------------------- applyLocalChange (backend.js:54-91)
  // One change request (a change table holding one change) encoded on the device with the author's previous change hash as
  // one more dependency, and applied from device memory (isLocal). out: the patch without the new change's hash in its
  // deps; binary: the plain change (the caller DEFLATEs one of 256 bytes or more). A change of 256 bytes or more is marked
  // to go out DEFLATEd (deflateOnExport). Errors leave the document unchanged, except "Unknown change" when the change
  // waits in the queue after the apply, which the reference also raises after the apply.
  void applyLocalChange(const u8* table, size_t len, bool wantPatch, PatchOut& out, std::string& binary);

  // ---------------------------------------------------------------- hash-graph queries (graph.cuh; new.js:1921-2028)
  // The dependency graph of the applied changes over change indexes, in application order, and their hashes. extendGraph()
  // adds the changes applied since the last query. For a change applied by applyChanges, its dependency indexes and author
  // come from the gate's own resolution: commit copies the batch's tables device to device (keepGraphInputs, no kernel),
  // and the query reads them back. Any other change (a loaded document's, or one applied before a reset of these inputs)
  // has its header parsed in the device arena and its dependency hashes resolved against `hashes` (parseChangeHeaders,
  // resolveChangeDeps, SaveChangeValKernel for the author). The lists below are appended on the host. The hashes come back
  // with them, so that getChanges resolves haveDeps and the heads on the host: a query over a current graph launches
  // nothing. reset() drops the graph; a clone builds its own.
  struct ChangeGraph {
    size_t known = 0;                                 // changes [0, known) are in the graph
    std::vector<u32> depBase{0}, deps;                // change i's dependencies in header order: deps[depBase[i], depBase[i + 1])
    std::vector<u32> depOwner, nextDependent;         // per entry k of deps: the change it belongs to; the next entry naming the same dependency
    std::vector<u32> firstDependent, lastDependent;   // per change: the first / last entry of deps that names it (EMPTY32: none)
    std::vector<std::vector<u32>> byActor;            // byActor[actor number][seq - 1] = change index (an actor's changes apply in seq order)
    std::vector<std::array<u8, 32>> hash;             // per change
    std::vector<u32> slots;                           // open addressing over the first 8 hash bytes: change index or EMPTY32
    template <class F> void eachDependent(u32 c, F f) const { for (u32 k = firstDependent[c]; k != EMPTY32; k = nextDependent[k]) f(depOwner[k]); }   // in application order
    void add(u32 c, const u32* dep, size_t nDep, u32 actor, const u8* h);   // change c = known, its dependencies, author, hash
    u32 find(const u8* h) const;                      // the change with hash h, or DEP_MISSING
  } graph;
  // What commit keeps of each batch for the graph: per batch entry applied flag, application rank, author's actor number,
  // dependency offsets; the dependency indexes (gate numbering: < first: applied before, else first + batch entry).
  struct GraphInputs {
    struct Batch { size_t first, B, D, numNew, offB, offBase, offD; };
    std::vector<Batch> batches; size_t usedB = 0, usedBase = 0, usedD = 0;
    DBuf<u8> applied; DBuf<u32> rank, actor, depBase, depIdx;
    void clear() { batches.clear(); usedB = usedBase = usedD = 0; }
  } graphInputs;
  void keepGraphInputs(ApplyCall& a);
  void extendGraph();
  void graphFromHeaders(size_t from, size_t to);
  void graphFromBatch(const GraphInputs::Batch& b);
  // Each query computes the hash graph of a loaded document first (new.js:1922, 2000, 2015) and times its device work in
  // spans[SPAN_GRAPH]. changesSince: getChanges(haveDeps) as change indexes in the order the reference returns them.
  void changesSince(const u8* haveDeps, size_t n, std::vector<u32>& out);
  bool changeIndexOf(const u8* hash, u32& idx);   // getChangeByHash: false for a hash that is not an applied change's
  void missingDeps(const u8* heads, size_t n, std::vector<std::array<u8, 32>>& out);   // getMissingDeps: sorted, without repeats
  bool hashByActor(const std::string& actor, u64 index, u8* out);   // the hash of actor's change seq = index + 1
  void lookupHashes(const u8* hs, size_t n, std::vector<u32>& idx);   // idx[i]: the applied change with hash hs[i], or DEP_MISSING
  DBuf<u8> graphQueries; DBuf<u32> graphIdx; DBuf<long long> graphVals;
 private:
  void lookupQueries(size_t n, size_t count, std::vector<u32>& idx);   // graphQueries[0, n) among hashes [0, count)
  void uploadCandidates(const u32* idx, size_t count);
};

}  // namespace amg
