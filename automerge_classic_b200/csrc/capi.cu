// amgpu — extern "C" surface (include/amgpu.h) over amg::Engine. The hash-graph queries (reference backend/new.js:1921-2028)
// are answered by the engine from its device hashes; only the change bytes they return come from the host arena copy.
#include "../../include/amgpu.h"
#include "engine_impl.cuh"

using namespace amg;

struct amg_patch { const u8* p; size_t len; };   // view into the engine's pinned patch buffer
struct amg_buffers { std::vector<std::string> items; };

struct amg_backend {
  Engine eng;
  explicit amg_backend(int dev) : eng(dev) {}

  // columnar.js:798-811 deflateChange: magic + checksum of the plain form, chunk type 2, raw DEFLATE of the body
  static std::string deflateChange(const std::string& plain) {
    ByteReader r((const u8*)plain.data(), 9, (u32)plain.size()); const u64 bodyLen = r.uleb();
    if (r.err || r.pos + bodyLen != plain.size()) throw amg::Error(AMG_ERR_INTERNAL, "deflateChange: malformed change");
    const std::string comp = amg::deflateRawBytes((const u8*)plain.data() + r.pos, (size_t)bodyLen);
    std::string out(plain, 0, 8); out.push_back(2); amg::put_uleb(out, comp.size());
    return out + comp;
  }
  std::string changeBytes(u32 idx) {
    eng.ensureHostMirror();
    if (const HostChange* o = eng.originalOf(idx)) return std::string((const char*)eng.hostArena.data() + o->off, o->len);
    const HostChange& c = eng.changes[idx];
    std::string plain((const char*)eng.hostArena.data() + c.off, c.len);
    return eng.exportsDeflated(idx) ? deflateChange(plain) : plain;
  }
};

namespace {
void setErr(amg_error* err, int code, const std::string& msg) {
  if (!err) return;
  err->code = code; snprintf(err->msg, sizeof(err->msg), "%s", msg.c_str());
}
// A failed call: the peeks it left pending are dropped, *err and (for an amg::Error) *failed are set, the code is returned
int fail(amg_error* err, int code, const char* msg, size_t* failed = nullptr, size_t failedAt = 0) {
  amg::drop_pending_peeks(); setErr(err, code, msg);
  if (failed) *failed = failedAt;
  return code;
}
// The body of an extern "C" call returning an error code; AMG_GUARD_FAILED also reports `source` (read after the throw)
// in *failed when the call fails with an amg::Error
#define AMG_GUARD_FAILED(failed, source, ...) \
  try { __VA_ARGS__ } catch (amg::Error& e) { return fail(err, e.code, e.what(), failed, source); } \
  catch (std::exception& e) { return fail(err, AMG_INTERNAL_ERROR, e.what()); }
#define AMG_GUARD(...) AMG_GUARD_FAILED(nullptr, 0, __VA_ARGS__)

// amg_init / amg_load / amg_clone: a new backend that `fill` completes, or nullptr with *err set (the backend is freed)
template <class F> amg_backend* construct(int device, amg_error* err, F fill) {
  try { std::unique_ptr<amg_backend> b(new amg_backend(device)); fill(*b); return b.release(); }
  catch (amg::Error& e) { fail(err, e.code, e.what()); }
  catch (std::exception& e) { fail(err, AMG_INTERNAL_ERROR, e.what()); }
  return nullptr;
}

// A list for the caller, filled by `fill`; freed if fill throws
template <class F> std::unique_ptr<amg_buffers> buffers(F fill) { std::unique_ptr<amg_buffers> l(new amg_buffers()); fill(l->items); return l; }
typedef std::vector<std::string> Items;

amg_patch* serialize(const PatchOut& p) { return new amg_patch{p.bytes, p.bytesLen}; }
}  // namespace

extern "C" {

amg_backend* amg_init(int cuda_device, amg_error* err) { return construct(cuda_device, err, [](amg_backend&) {}); }
void amg_free(amg_backend* b) { delete b; }
amg_backend* amg_load(int cuda_device, const uint8_t* data, size_t len, amg_error* err) {
  return construct(cuda_device, err, [&](amg_backend& b) { b.eng.loadDocument(data, len); });
}
int amg_reset(amg_backend* b, amg_error* err) { AMG_GUARD(b->eng.reset(); return 0;) }
int amg_reserve(amg_backend* b, size_t arena_bytes, amg_error* err) { AMG_GUARD(b->eng.hostArena.reserve(arena_bytes); b->eng.arena.ensure(b->eng.ctx, arena_bytes + 64, b->eng.arenaLen); return 0;) }

amg_backend* amg_clone(amg_backend* src, amg_error* err) {
  return construct(src->eng.ctx.device, err, [&](amg_backend& b) {
    Engine& d = b.eng; Engine& s = src->eng; Ctx& c = d.ctx;
    sync(s.ctx); s.ensureHostMirror();
    d.hostArena.assign(s.hostArena); d.arenaLen = s.arenaLen; d.arena.ensure(c, s.arenaLen + 64); d2d(c, d.arena.p, s.arena.p, s.arenaLen);
    d.numApplied = s.numApplied; d.hashes.ensure(c, s.numApplied * 32 + 64); d2d(c, d.hashes.p, s.hashes.p, s.numApplied * 32);
    d.numRows = s.numRows; d.doc.copyFrom(c, s.doc, s.numRows);
    d.numSucc = s.numSucc; d.succOff.ensure(c, s.numRows + 2); d2d(c, d.succOff.p, s.succOff.p, (s.numRows + 1) * 4); d.succ.ensure(c, s.numSucc + 1); d2d(c, d.succ.p, s.succ.p, s.numSucc * 8);
    d.lastChange.ensure(c, s.st.actorIds.size() + 1); d2d(c, d.lastChange.p, s.lastChange.p, s.st.actorIds.size() * 4);
    d.st = s.st; d.changes = s.changes; d.deflatedOriginal = s.deflatedOriginal; d.deflateOnExport = s.deflateOnExport; d.loaded = s.loaded;
    d.unknownCols = s.unknownCols; d.queue = s.queue; d.queueOriginal = s.queueOriginal;
    while (d.actorCap < 2 * (d.st.actorIds.size() + 16)) d.actorCap *= 2;
    d.actorSlots.ensure(c, d.actorCap); d.rebuildActorTable();
    sync(c);
  });
}

int amg_apply_changes(amg_backend* b, const uint8_t* const* bufs, const size_t* lens, size_t n, int is_local, int want_patch, amg_patch** out, amg_error* err) {
  AMG_GUARD(PatchOut p; b->eng.applyChanges(bufs, lens, n, nullptr, nullptr, is_local != 0, want_patch != 0, p);
            if (out) *out = want_patch ? serialize(p) : nullptr; return 0;)
}
int amg_apply_changes_packed(amg_backend* b, const uint8_t* blob, const uint64_t* offsets, size_t n, int is_local, int want_patch, amg_patch** out, amg_error* err) {
  AMG_GUARD(amg::HostClock whole; { PatchOut p; b->eng.applyChanges(nullptr, nullptr, n, blob, (const u64*)offsets, is_local != 0, want_patch != 0, p);
            if (out) *out = want_patch ? serialize(p) : nullptr; } b->eng.trace.ms[23] = whole.ms(); return 0;)   // [23]: the whole call as the ABI sees it
}
int amg_get_patch(amg_backend* b, amg_patch** out, amg_error* err) {
  AMG_GUARD(PatchOut p; b->eng.getPatch(p); *out = serialize(p); return 0;)
}
int amg_get_state(amg_backend* b, amg_patch** out, amg_error* err) {
  AMG_GUARD(PatchOut p; b->eng.fillPatchHeader(p); b->eng.finishPatch(p); *out = serialize(p); return 0;)
}
const uint8_t* amg_patch_bytes(const amg_patch* p, size_t* len) { *len = p->len; return p->p; }
void amg_patch_free(amg_patch* p) { delete p; }
const uint8_t* amg_arena(amg_backend* b, size_t* len) {
  try { b->eng.ensureHostMirror(); } catch (...) { amg::drop_pending_peeks(); *len = 0; return nullptr; }
  *len = b->eng.hostArena.size(); return b->eng.hostArena.data();
}

size_t amg_buffers_count(const amg_buffers* l) { return l->items.size(); }
const uint8_t* amg_buffers_get(const amg_buffers* l, size_t i, size_t* len) { *len = l->items[i].size(); return (const uint8_t*)l->items[i].data(); }
void amg_buffers_free(amg_buffers* l) { delete l; }
void amg_free_mem(void* p) { free(p); }

int amg_get_heads(amg_backend* b, amg_buffers** out, amg_error* err) {
  AMG_GUARD(*out = buffers([&](Items& l) { for (auto& h : b->eng.st.heads) l.emplace_back((const char*)h.data(), 32); }).release(); return 0;)
}

// new.js:2033-2055
int amg_save(amg_backend* b, amg_buffers** out, amg_error* err) {
  AMG_GUARD(*out = buffers([&](Items& l) { l.emplace_back(); b->eng.saveDocument(l.back()); }).release(); return 0;)
}

// new.js:1921-1973
int amg_get_changes(amg_backend* b, const uint8_t* have_deps, size_t n, amg_buffers** out, amg_error* err) {
  AMG_GUARD(
    std::vector<u32> idx; b->eng.changesSince(have_deps, n, idx);
    *out = buffers([&](Items& l) { for (u32 i : idx) l.push_back(b->changeBytes(i)); }).release(); return 0;)
}
// sync.js:234-238 makeBloomFilter: Bloom filter over the hashes of getChanges(last_sync), built on the device
int amg_sync_bloom(amg_backend* b, const uint8_t* last_sync, size_t n, amg_buffers** out, amg_error* err) {
  AMG_GUARD(
    Engine& e = b->eng; e.computeHashGraph();   // the hashes of a loaded document (new.js:1922)
    *out = buffers([&](Items& l) {
      l.emplace_back();
      if (n == 0) e.syncBloom(nullptr, e.numApplied, l.back());   // every applied change: no graph walk needed
      else { std::vector<u32> idx; e.changesSince(last_sync, n, idx); e.syncBloom(idx.data(), idx.size(), l.back()); }
    }).release(); return 0;)
}
// sync.js:246-306 getChangesToSend for a non-empty `have`
int amg_sync_changes_to_send(amg_backend* b, const uint8_t* last_sync, size_t n_last, const amg_bloom* filters, size_t n_filters,
                             const uint8_t* need, size_t n_need, amg_buffers** out_changes, amg_buffers** out_hashes, amg_error* err) {
  AMG_GUARD(
    Engine& e = b->eng; e.computeHashGraph();
    std::vector<u32> cand; if (n_last > 0) e.changesSince(last_sync, n_last, cand);
    const u32* idx = n_last > 0 ? cand.data() : nullptr; const size_t count = n_last > 0 ? cand.size() : e.numApplied;
    std::vector<Engine::BloomSpec> fs(n_filters);
    for (size_t i = 0; i < n_filters; i++) fs[i] = Engine::BloomSpec{filters[i].num_entries, filters[i].num_probes, filters[i].bits, filters[i].bits_len};
    std::vector<u8> send; e.syncChangesToSend(idx, count, fs, send);
    // sync.js:291-305: first the needed changes that are not candidates (unknown ones are skipped), then, in candidate
    // order, the candidates that were marked or are needed
    std::vector<u32> outIdx;
    if (n_need > 0) {
      std::vector<u32> needIdx; e.spans.resume(SPAN_SYNC); e.lookupHashes(need, n_need, needIdx); e.spans.stop();
      std::vector<u32> posOf(e.numApplied, EMPTY32);   // change index -> candidate position
      for (size_t i = 0; i < count; i++) posOf[idx ? idx[i] : i] = (u32)i;
      for (u32 c : needIdx) {
        if (c == DEP_MISSING) continue;
        if (posOf[c] != EMPTY32) send[posOf[c]] = 1; else outIdx.push_back(c);
      }
    }
    for (size_t i = 0; i < count; i++) if (send[i]) outIdx.push_back(idx ? idx[i] : (u32)i);
    auto lh = buffers([&](Items& l) { l.emplace_back(); e.gatherHashes(outIdx, l.back()); });
    auto lc = buffers([&](Items& l) { for (u32 i : outIdx) l.push_back(b->changeBytes(i)); });
    *out_changes = lc.release(); *out_hashes = lh.release(); return 0;)
}
float amg_last_sync_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_SYNC]; }
// columnar.js:770-776 decodeChange over n change containers, into one change table
int amg_decode_changes(amg_backend* b, const uint8_t* blob, const uint64_t* offsets, size_t n, amg_buffers** out, size_t* failed_index, amg_error* err) {
  if (failed_index) *failed_index = 0;
  AMG_GUARD_FAILED(failed_index, b->eng.decodeFailed,
    *out = buffers([&](Items& l) { l.emplace_back(); b->eng.decodeChanges(blob, (const u64*)offsets, n, false, l.back()); }).release(); return 0;)
}
// the same for every applied change, in getAllChanges order (new.js:1925-1927), read from device memory
int amg_decode_history(amg_backend* b, amg_buffers** out, amg_error* err) {
  AMG_GUARD(
    b->eng.computeHashGraph();   // (new.js:1922) before the change count is taken
    *out = buffers([&](Items& l) { l.emplace_back(); b->eng.decodeChanges(nullptr, nullptr, b->eng.changes.size(), true, l.back()); }).release(); return 0;)
}
float amg_last_decode_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_DECODE]; }
// columnar.js:710-739 encodeChange over the changes of a change table: plain changes from the device, the ones of 256 bytes
// or more DEFLATEd here (columnar.js:738), over a few host threads when there are many
int amg_encode_changes(amg_backend* b, const uint8_t* table, size_t table_len, amg_buffers** out_changes, amg_buffers** out_hashes,
                       size_t* failed_index, amg_error* err) {
  if (failed_index) *failed_index = 0;
  AMG_GUARD_FAILED(failed_index, b->eng.encodeFailed,
    std::string bytes, hs; std::vector<u64> offs;
    b->eng.encodeChanges(table, table_len, bytes, offs, hs);
    auto lc = buffers([&](Items& l) {
      const size_t n = offs.size() - 1; l.resize(n);
      auto fill = [&](size_t from, size_t to) {
        for (size_t i = from; i < to; i++) {
          const u64 len = offs[i + 1] - offs[i];
          if (len >= 256) l[i] = amg_backend::deflateChange(std::string(bytes, offs[i], len)); else l[i].assign(bytes, offs[i], len);
        }
      };
      const size_t nThreads = std::min<size_t>(std::max(1u, std::thread::hardware_concurrency()), std::min<size_t>(16, n / 4096 + 1));
      if (nThreads <= 1) fill(0, n);
      else {
        std::vector<std::thread> th; const size_t per = (n + nThreads - 1) / nThreads;
        for (size_t t = 0; t < nThreads; t++) th.emplace_back(fill, std::min(n, t * per), std::min(n, (t + 1) * per));
        for (auto& x : th) x.join();
      }
    });
    auto lh = buffers([&](Items& l) { l.push_back(std::move(hs)); });
    *out_changes = lc.release(); *out_hashes = lh.release(); return 0;)
}
float amg_last_encode_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_ENCODE]; }
// src/automerge.js:105-118 getHistory's snapshots: getPatch(loadChanges(init(), getAllChanges()[0, k))) for every k
int amg_get_history_patches(amg_backend* b, const uint64_t* prefix_lens, size_t n, amg_buffers** out, amg_error* err) {
  AMG_GUARD(*out = buffers([&](Items& l) { b->eng.historyPatches((const u64*)prefix_lens, n, l); }).release(); return 0;)
}
float amg_last_history_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_HISTORY]; }
// new.js:1979-1997: the changes in their order from Engine::changesAddedFrom (no host hash graph is built)
int amg_get_changes_added(amg_backend* bn, amg_backend* bo, amg_buffers** out, amg_error* err) {
  AMG_GUARD(
    std::vector<u32> idx; bo->eng.changesAddedFrom(bn->eng, idx);
    *out = buffers([&](Items& l) { for (u32 i : idx) l.push_back(bn->changeBytes(i)); }).release(); return 0;)
}
// src/automerge.js:61-67 merge(local, remote): applyChanges(local, getChangesAdded(local, remote)), the bytes device to device
int amg_merge(amg_backend* dst, amg_backend* src, int want_patch, amg_patch** out, amg_error* err) {
  AMG_GUARD(PatchOut p; dst->eng.mergeFrom(src->eng, want_patch != 0, p);
            if (out) *out = want_patch ? serialize(p) : nullptr; return 0;)
}
float amg_last_merge_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_MERGE]; }
// backend/backend.js:54-91 applyLocalChange: encoded and applied on the device; the returned change DEFLATEd here when
// 256 bytes or more (columnar.js:738), as amg_encode_changes returns it
int amg_apply_local_change(amg_backend* b, const uint8_t* table, size_t table_len, int want_patch, amg_patch** out, amg_buffers** out_change, amg_error* err) {
  AMG_GUARD(PatchOut p; std::string plain; b->eng.applyLocalChange(table, table_len, want_patch != 0, p, plain);
            auto lc = buffers([&](Items& l) { l.push_back(plain.size() >= 256 ? amg_backend::deflateChange(plain) : plain); });
            if (out) *out = want_patch ? serialize(p) : nullptr;
            *out_change = lc.release(); return 0;)
}
float amg_last_local_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_LOCAL]; }
// new.js:1999-2002
int amg_get_change_by_hash(amg_backend* b, const uint8_t hash[32], amg_buffers** out, amg_error* err) {
  AMG_GUARD(u32 idx = 0; const bool found = b->eng.changeIndexOf(hash, idx);
            *out = buffers([&](Items& l) { if (found) l.push_back(b->changeBytes(idx)); }).release(); return 0;)
}
// new.js:2014-2028
int amg_get_missing_deps(amg_backend* b, const uint8_t* heads, size_t n, amg_buffers** out, amg_error* err) {
  AMG_GUARD(
    std::vector<std::array<u8, 32>> missing; b->eng.missingDeps(heads, n, missing);
    *out = buffers([&](Items& l) { for (auto& h : missing) l.emplace_back((const char*)h.data(), 32); }).release(); return 0;)
}
float amg_last_graph_ms(amg_backend* b) { return b->eng.spans.ms[SPAN_GRAPH]; }
int amg_clock_of(amg_backend* b, const uint8_t* actor, size_t actor_len, uint64_t* seq_out, amg_error* err) {
  AMG_GUARD(std::string a((const char*)actor, actor_len); *seq_out = 0; Engine& e = b->eng;
            for (size_t i = 0; i < e.st.actorIds.size(); i++) if (e.st.actorIds[i] == a) *seq_out = e.st.clock[i]; return 0;)
}
int amg_hash_by_actor(amg_backend* b, const uint8_t* actor, size_t actor_len, uint64_t index, uint8_t hash_out[32], int* found, amg_error* err) {
  AMG_GUARD(*found = b->eng.hashByActor(std::string((const char*)actor, actor_len), index, hash_out) ? 1 : 0; return 0;)
}

int amg_last_timings(amg_backend* b, float* ms_out, int n) { for (int i = 0; i < n && i < 24; i++) ms_out[i] = b->eng.trace.ms[i]; return 0; }
size_t amg_debug_marks(amg_backend* b, char* buf, size_t cap) {
  std::string s; for (auto& m : b->eng.trace.marks) { char t[96]; snprintf(t, sizeof t, "%s=%.3f ", m.first, m.second); s += t; }
  if (cap) { snprintf(buf, cap, "%s", s.c_str()); } return s.size();
}
uint64_t amg_kernel_launches(amg_backend* b) { return b->eng.ctx.launches; }

int amg_debug_dump_ops(amg_backend* b, uint64_t** rows_out, size_t* n, uint64_t** succ_out, size_t* m, amg_error* err) {
  AMG_GUARD(
    Engine& e = b->eng; const size_t N = e.numRows, S = e.numSucc;
    std::vector<u64> id(N), obj(N), key(N), succ(S); std::vector<u32> flags(N), soff(N + 1), ksl(N);
    d2h(e.ctx, id.data(), e.doc.id.p, N * 8); d2h(e.ctx, obj.data(), e.doc.obj.p, N * 8); d2h(e.ctx, key.data(), e.doc.key.p, N * 8);
    d2h(e.ctx, flags.data(), e.doc.flags.p, N * 4); d2h(e.ctx, ksl.data(), e.doc.keyStrLen.p, N * 4); d2h(e.ctx, soff.data(), e.succOff.p, (N + 1) * 4); d2h(e.ctx, succ.data(), e.succ.p, S * 8); sync(e.ctx);
    u64* r = (u64*)malloc(sizeof(u64) * 8 * (N + 1)); u64* s = (u64*)malloc(sizeof(u64) * 2 * (S + 1));
    for (size_t i = 0; i < N; i++) {
      u64* o = r + 8 * i; const u64 none = ~0ULL;
      o[0] = obj[i] ? id_ctr(obj[i]) : none; o[1] = obj[i] ? id_actor(obj[i]) : none; o[2] = id_ctr(id[i]); o[3] = id_actor(id[i]);
      const bool list = ksl[i] == NULL32;
      o[4] = list ? id_ctr(key[i]) : none; o[5] = (list && key[i]) ? id_actor(key[i]) : none; o[6] = flags[i]; o[7] = soff[i + 1] - soff[i];
    }
    for (size_t i = 0; i < S; i++) { s[2 * i] = id_ctr(succ[i]); s[2 * i + 1] = id_actor(succ[i]); }
    *rows_out = (uint64_t*)r; *n = N; *succ_out = (uint64_t*)s; *m = S; return 0;)
}

int amg_debug_decode(amg_backend* b, const uint8_t* blob, const uint64_t* offsets, size_t n, uint8_t* hashes_out, uint32_t* n_ops_out, uint32_t** rows_out, size_t* total_ops, size_t* total_preds, amg_error* err) {
  AMG_GUARD(b->eng.decodeRaw(blob, (const u64*)offsets, n, hashes_out, n_ops_out, rows_out, total_ops, total_preds); return 0;)
}
int amg_debug_decode_column(amg_backend* b, const uint8_t* bytes, size_t len, int kind, size_t n, int parallel, int64_t* out, amg_error* err) {
  AMG_GUARD(return b->eng.debugDecodeColumn(bytes, len, kind, n, parallel != 0, (long long*)out);)
}
int amg_bench_decode(amg_backend* b, int iters, float* ms_sha, float* ms_parse, float* ms_decode, uint64_t* algo_bytes, amg_error* err) {
  AMG_GUARD(u64 bytes = 0; b->eng.benchDecode(iters, ms_sha, ms_parse, ms_decode, &bytes); *algo_bytes = bytes; return 0;)
}
}  // extern "C"
