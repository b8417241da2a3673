// N-API addon: binds the C ABI of libamgpu.so (include/amgpu.h) for Node. This is the thin layer north_star asks for:
// the host stays JavaScript, every Backend function of the reference (backend/index.js:1-8, backend/backend.js) lands
// on one amg_* call. The JS side (js/index.js) wraps it into the module shape Automerge.setDefaultBackend() expects
// (src/automerge.js:147-149) and inflates the flat patch (js/inflate_patch.js).
//
// Build (on a machine with Node): cd addon && node-gyp rebuild   (binding.gyp links ../automerge_classic_b200/libamgpu.so)
// Node / node_api.h are not present in the build image of this repository: the file is kept compiling against a minimal
// declaration stub (addon/stub/node_api.h; `make -C addon check`) and is otherwise exercised through the Python twin of
// the same calls (automerge_classic_b200/engine.py), which is what the parity tests drive.
#include <node_api.h>
#include <cstring>
#include <string>
#include <vector>
#include "amgpu.h"

namespace {

// The reference throws RangeError / TypeError / Error synchronously (backend/new.js:1256, 1573, ...); amg_error carries
// the reference's message text.
napi_value throwAmg(napi_env env, const amg_error& err) {
  if (err.code == AMG_RANGE_ERROR) napi_throw_range_error(env, nullptr, err.msg);
  else if (err.code == AMG_TYPE_ERROR) napi_throw_type_error(env, nullptr, err.msg);
  else napi_throw_error(env, nullptr, err.msg);
  return nullptr;
}
// S of @types/automerge/index.d.ts:186-188: an external holding the amg_backend*; released by Backend.free (backend.js:16-19)
// or, failing that, when the external is garbage collected
struct Holder { amg_backend* b; };
void finalizeBackend(napi_env, void* data, void*) { Holder* h = static_cast<Holder*>(data); if (h->b) amg_free(h->b); delete h; }
napi_value wrapBackend(napi_env env, amg_backend* b) {
  napi_value out; napi_create_external(env, new Holder{b}, finalizeBackend, nullptr, &out); return out;
}
bool getHolder(napi_env env, napi_value v, Holder** out) {
  void* p = nullptr;
  if (napi_get_value_external(env, v, &p) != napi_ok || !p) { napi_throw_type_error(env, nullptr, "not a backend state"); return false; }
  *out = static_cast<Holder*>(p); return true;
}
bool getBackend(napi_env env, napi_value v, amg_backend** out) {
  Holder* h; if (!getHolder(env, v, &h)) return false;
  if (!h->b) { napi_throw_error(env, nullptr, "backend state has been freed"); return false; }
  *out = h->b; return true;
}
bool getBytes(napi_env env, napi_value v, const uint8_t** data, size_t* len) {   // Uint8Array / Buffer, no copy
  bool isTyped = false; napi_is_typedarray(env, v, &isTyped);
  if (!isTyped) { napi_throw_type_error(env, nullptr, "expected a Uint8Array"); return false; }
  napi_typedarray_type type; napi_value ab; size_t off; void* p = nullptr;
  if (napi_get_typedarray_info(env, v, &type, len, &p, &ab, &off) != napi_ok || type != napi_uint8_array) { napi_throw_type_error(env, nullptr, "expected a Uint8Array"); return false; }
  *data = static_cast<const uint8_t*>(p); return true;
}
napi_value bytesToUint8Array(napi_env env, const uint8_t* p, size_t len) {
  napi_value ab, out; void* copy = nullptr;
  napi_create_arraybuffer(env, len, &copy, &ab); if (len) memcpy(copy, p, len);
  napi_create_typedarray(env, napi_uint8_array, len, ab, 0, &out); return out;
}
napi_value patchToJs(napi_env env, amg_patch* patch) {   // flat patch (layout: amgpu.h) -> Uint8Array; nested Patch is built in JS
  if (!patch) { napi_value u; napi_get_undefined(env, &u); return u; }
  size_t len = 0; const uint8_t* bytes = amg_patch_bytes(patch, &len);
  napi_value out = bytesToUint8Array(env, bytes, len);
  amg_patch_free(patch); return out;
}
napi_value buffersToJs(napi_env env, amg_buffers* l) {
  const size_t n = amg_buffers_count(l); napi_value arr; napi_create_array_with_length(env, n, &arr);
  for (size_t i = 0; i < n; i++) { size_t len = 0; const uint8_t* p = amg_buffers_get(l, i, &len); napi_set_element(env, arr, (uint32_t)i, bytesToUint8Array(env, p, len)); }
  amg_buffers_free(l); return arr;
}
bool getArgs(napi_env env, napi_callback_info info, size_t want, napi_value* argv) {
  size_t argc = want; if (napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr) != napi_ok || argc < want) { napi_throw_type_error(env, nullptr, "missing argument"); return false; }
  return true;
}
int deviceFromEnv() { const char* d = getenv("AMG_DEVICE"); return d ? atoi(d) : 0; }

// Backend.init() — backend/backend.js:8-10
napi_value Init(napi_env env, napi_callback_info) {
  amg_error err; amg_backend* b = amg_init(deviceFromEnv(), &err);
  return b ? wrapBackend(env, b) : throwAmg(env, err);
}
// Backend.load(data) — backend/backend.js:104-107
napi_value Load(napi_env env, napi_callback_info info) {
  napi_value argv[1]; if (!getArgs(env, info, 1, argv)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[0], &p, &len)) return nullptr;
  amg_error err; amg_backend* b = amg_load(deviceFromEnv(), p, len, &err);
  return b ? wrapBackend(env, b) : throwAmg(env, err);
}
// Backend.clone — backend/backend.js:12-14
napi_value Clone(napi_env env, napi_callback_info info) {
  napi_value argv[1]; amg_backend* b; if (!getArgs(env, info, 1, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  amg_error err; amg_backend* c = amg_clone(b, &err);
  return c ? wrapBackend(env, c) : throwAmg(env, err);
}
// applyChanges(state, Uint8Array[], isLocal, wantPatch) — backend/backend.js:27-32 (isLocal: :84; wantPatch false = loadChanges :116-121)
napi_value ApplyChanges(napi_env env, napi_callback_info info) {
  napi_value argv[4]; amg_backend* b; if (!getArgs(env, info, 4, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  bool isArray = false; napi_is_array(env, argv[1], &isArray);
  if (!isArray) { napi_throw_type_error(env, nullptr, "applyChanges takes an array of Uint8Arrays"); return nullptr; }   // new.js:1798-1803
  uint32_t n = 0; napi_get_array_length(env, argv[1], &n);
  std::vector<const uint8_t*> bufs(n); std::vector<size_t> lens(n);
  for (uint32_t i = 0; i < n; i++) {                       // Uint8Array[] -> pointers, no copy on the JS side
    napi_value el; napi_get_element(env, argv[1], i, &el);
    if (!getBytes(env, el, &bufs[i], &lens[i])) return nullptr;
  }
  bool isLocal = false, wantPatch = true; napi_get_value_bool(env, argv[2], &isLocal); napi_get_value_bool(env, argv[3], &wantPatch);
  amg_patch* patch = nullptr; amg_error err;
  if (amg_apply_changes(b, bufs.data(), lens.data(), n, isLocal, wantPatch, &patch, &err)) return throwAmg(env, err);
  return patchToJs(env, patch);
}
// Backend.getPatch — backend/backend.js:127-129
napi_value GetPatch(napi_env env, napi_callback_info info) {
  napi_value argv[1]; amg_backend* b; if (!getArgs(env, info, 1, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  amg_patch* patch = nullptr; amg_error err;
  if (amg_get_patch(b, &patch, &err)) return throwAmg(env, err);
  return patchToJs(env, patch);
}
typedef int (*ListFn)(amg_backend*, amg_buffers**, amg_error*);
napi_value listCall(napi_env env, napi_callback_info info, ListFn fn, bool first) {
  napi_value argv[1]; amg_backend* b; if (!getArgs(env, info, 1, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  amg_buffers* l = nullptr; amg_error err;
  if (fn(b, &l, &err)) return throwAmg(env, err);
  napi_value arr = buffersToJs(env, l);
  if (!first) return arr;
  napi_value el; napi_get_element(env, arr, 0, &el); return el;
}
// Backend.save — backend/backend.js:93-95; Backend.getHeads — :135-137 (hashes as 32-byte arrays; hex in JS)
napi_value Save(napi_env env, napi_callback_info info) { return listCall(env, info, amg_save, true); }
napi_value GetHeads(napi_env env, napi_callback_info info) { return listCall(env, info, amg_get_heads, false); }
// hashes: Uint8Array of n x 32 bytes
napi_value hashListCall(napi_env env, napi_callback_info info, int (*fn)(amg_backend*, const uint8_t*, size_t, amg_buffers**, amg_error*)) {
  napi_value argv[2]; amg_backend* b; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[1], &p, &len)) return nullptr;
  amg_buffers* l = nullptr; amg_error err;
  if (fn(b, p, len / 32, &l, &err)) return throwAmg(env, err);
  return buffersToJs(env, l);
}
// Backend.getChanges(haveDeps) — backend/backend.js:151-156; getMissingDeps(heads) — :190-192
napi_value GetChanges(napi_env env, napi_callback_info info) { return hashListCall(env, info, amg_get_changes); }
napi_value GetMissingDeps(napi_env env, napi_callback_info info) { return hashListCall(env, info, amg_get_missing_deps); }
// Backend.getChangesAdded(old, new) — backend/backend.js:166-168
napi_value GetChangesAdded(napi_env env, napi_callback_info info) {
  napi_value argv[2]; amg_backend *older, *newer; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &older) || !getBackend(env, argv[1], &newer)) return nullptr;
  amg_buffers* l = nullptr; amg_error err;
  if (amg_get_changes_added(newer, older, &l, &err)) return throwAmg(env, err);
  return buffersToJs(env, l);
}
// Backend.getChangeByHash — backend/backend.js:176-178 (undefined when unknown)
napi_value GetChangeByHash(napi_env env, napi_callback_info info) {
  napi_value argv[2]; amg_backend* b; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[1], &p, &len) || len != 32) { napi_throw_type_error(env, nullptr, "expected a 32-byte hash"); return nullptr; }
  amg_buffers* l = nullptr; amg_error err;
  if (amg_get_change_by_hash(b, p, &l, &err)) return throwAmg(env, err);
  napi_value arr = buffersToJs(env, l), el; uint32_t n = 0; napi_get_array_length(env, arr, &n);
  if (n == 0) { napi_get_undefined(env, &el); return el; }
  napi_get_element(env, arr, 0, &el); return el;
}
// state needed by applyLocalChange in JS (backend/backend.js:54-91): clock[actor], hashesByActor[actor][index]
napi_value ClockOf(napi_env env, napi_callback_info info) {
  napi_value argv[2]; amg_backend* b; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[1], &p, &len)) return nullptr;
  uint64_t seq = 0; amg_error err; if (amg_clock_of(b, p, len, &seq, &err)) return throwAmg(env, err);
  napi_value out; napi_create_double(env, (double)seq, &out); return out;
}
napi_value HashByActor(napi_env env, napi_callback_info info) {
  napi_value argv[3]; amg_backend* b; if (!getArgs(env, info, 3, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[1], &p, &len)) return nullptr;
  double index = 0; napi_get_value_double(env, argv[2], &index);
  uint8_t hash[32]; int found = 0; amg_error err;
  if (amg_hash_by_actor(b, p, len, (uint64_t)index, hash, &found, &err)) return throwAmg(env, err);
  if (!found) { napi_value u; napi_get_undefined(env, &u); return u; }
  return bytesToUint8Array(env, hash, 32);
}
// syncBloom(state, lastSync) — sync.js:234-238 makeBloomFilter(backend, lastSync).bloom; lastSync: Uint8Array of n x 32 bytes
napi_value SyncBloom(napi_env env, napi_callback_info info) {
  napi_value arr = hashListCall(env, info, amg_sync_bloom), el; if (!arr) return nullptr;
  napi_get_element(env, arr, 0, &el); return el;
}
// syncChangesToSend(state, lastSync, filters, need) — sync.js:246-306 getChangesToSend for a non-empty `have`. lastSync, need:
// Uint8Array of n x 32 bytes; filters: array of parsed Bloom filters {numEntries, numProbes, bits: Uint8Array}. Returns
// [changes, hashes]: the changes to send in the reference's order, and one Uint8Array with their 32-byte hashes back to
// back (to filter sentHashes with).
napi_value SyncChangesToSend(napi_env env, napi_callback_info info) {
  napi_value argv[4]; amg_backend* b; if (!getArgs(env, info, 4, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  const uint8_t *last, *need; size_t lastLen, needLen;
  if (!getBytes(env, argv[1], &last, &lastLen) || !getBytes(env, argv[3], &need, &needLen)) return nullptr;
  bool isArray = false; napi_is_array(env, argv[2], &isArray);
  if (!isArray) { napi_throw_type_error(env, nullptr, "filters must be an array"); return nullptr; }
  uint32_t n = 0; napi_get_array_length(env, argv[2], &n);
  std::vector<amg_bloom> filters(n);
  for (uint32_t i = 0; i < n; i++) {
    napi_value f, v; napi_get_element(env, argv[2], i, &f);
    napi_get_named_property(env, f, "numEntries", &v); if (napi_get_value_uint32(env, v, &filters[i].num_entries) != napi_ok) { napi_throw_type_error(env, nullptr, "numEntries must be a number"); return nullptr; }
    napi_get_named_property(env, f, "numProbes", &v); if (napi_get_value_uint32(env, v, &filters[i].num_probes) != napi_ok) { napi_throw_type_error(env, nullptr, "numProbes must be a number"); return nullptr; }
    napi_get_named_property(env, f, "bits", &v); if (!getBytes(env, v, &filters[i].bits, &filters[i].bits_len)) return nullptr;
  }
  amg_buffers *changes = nullptr, *hashes = nullptr; amg_error err;
  if (amg_sync_changes_to_send(b, last, lastLen / 32, filters.data(), n, need, needLen / 32, &changes, &hashes, &err)) return throwAmg(env, err);
  napi_value out, hs; napi_create_array_with_length(env, 2, &out);
  napi_get_element(env, buffersToJs(env, hashes), 0, &hs);
  napi_set_element(env, out, 0, buffersToJs(env, changes)); napi_set_element(env, out, 1, hs);
  return out;
}
// the per-process backend handle decodeChanges and encodeChanges run on (created on first use)
amg_backend* codecBackend(amg_error* err) {
  static amg_backend* codec = nullptr;
  if (!codec) codec = amg_init(deviceFromEnv(), err);
  return codec;
}
// the reference's error class and message, with the index of the failing change as `failedIndex`
napi_value throwFailed(napi_env env, const amg_error& err, size_t failed) {
  napi_value msg, e, idx; napi_create_string_utf8(env, err.msg, NAPI_AUTO_LENGTH, &msg);
  if (err.code == AMG_RANGE_ERROR) napi_create_range_error(env, nullptr, msg, &e);
  else if (err.code == AMG_TYPE_ERROR) napi_create_type_error(env, nullptr, msg, &e);
  else napi_create_error(env, nullptr, msg, &e);
  napi_create_double(env, (double)failed, &idx); napi_set_named_property(env, e, "failedIndex", idx);
  napi_throw(env, e); return nullptr;
}
// decodeChanges(Uint8Array[]) — columnar.js:770-776 decodeChange of every entry (one change container each), in one call on
// a per-process backend handle. Returns the change table (layout: amgpu.h) as one Uint8Array; an error carries the index of
// the failing change as `failedIndex`.
napi_value DecodeChanges(napi_env env, napi_callback_info info) {
  napi_value argv[1]; if (!getArgs(env, info, 1, argv)) return nullptr;
  bool isArray = false; napi_is_array(env, argv[0], &isArray);
  if (!isArray) { napi_throw_type_error(env, nullptr, "decodeChanges takes an array of Uint8Arrays"); return nullptr; }
  uint32_t n = 0; napi_get_array_length(env, argv[0], &n);
  std::string blob; std::vector<uint64_t> offsets(n + 1, 0);
  for (uint32_t i = 0; i < n; i++) {
    napi_value el; napi_get_element(env, argv[0], i, &el);
    const uint8_t* p; size_t len; if (!getBytes(env, el, &p, &len)) return nullptr;
    blob.append(reinterpret_cast<const char*>(p), len); offsets[i + 1] = blob.size();
  }
  amg_error err; amg_backend* decoder = codecBackend(&err);
  if (!decoder) return throwAmg(env, err);
  amg_buffers* l = nullptr; size_t failed = 0;
  if (amg_decode_changes(decoder, reinterpret_cast<const uint8_t*>(blob.data()), offsets.data(), n, &l, &failed, &err)) return throwFailed(env, err, failed);
  napi_value el; napi_get_element(env, buffersToJs(env, l), 0, &el); return el;
}
// encodeChanges(Uint8Array) — columnar.js:710-739 encodeChange of every change of a change table (layout: amgpu.h), in one
// call on the same per-process backend handle. Returns {changes: Uint8Array[], hashes: Uint8Array (n x 32 bytes)}; an error
// carries the index of the failing change as `failedIndex`.
napi_value EncodeChanges(napi_env env, napi_callback_info info) {
  napi_value argv[1]; if (!getArgs(env, info, 1, argv)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[0], &p, &len)) return nullptr;
  amg_error err; amg_backend* encoder = codecBackend(&err);
  if (!encoder) return throwAmg(env, err);
  amg_buffers *changes = nullptr, *hashes = nullptr; size_t failed = 0;
  if (amg_encode_changes(encoder, p, len, &changes, &hashes, &failed, &err)) return throwFailed(env, err, failed);
  napi_value out, hs; napi_create_object(env, &out);
  napi_get_element(env, buffersToJs(env, hashes), 0, &hs);
  napi_set_named_property(env, out, "changes", buffersToJs(env, changes)); napi_set_named_property(env, out, "hashes", hs);
  return out;
}
// decodeHistory(state) — decodeChanges(getAllChanges(state)), read from device memory: the change table as one Uint8Array
napi_value DecodeHistory(napi_env env, napi_callback_info info) { return listCall(env, info, amg_decode_history, true); }
// historyPatches(state, prefixLengths) — src/automerge.js:105-118 getHistory's snapshots: for every k of the array, the flat
// patch (layout: amgpu.h) of getPatch(loadChanges(init(), getAllChanges(state).slice(0, k))), one Uint8Array each
napi_value HistoryPatches(napi_env env, napi_callback_info info) {
  napi_value argv[2]; amg_backend* b; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  bool isArray = false; napi_is_array(env, argv[1], &isArray);
  if (!isArray) { napi_throw_type_error(env, nullptr, "prefixLengths must be an array of numbers"); return nullptr; }
  uint32_t n = 0; napi_get_array_length(env, argv[1], &n);
  std::vector<uint64_t> lens(n);
  for (uint32_t i = 0; i < n; i++) {
    napi_value el; double k = 0; napi_get_element(env, argv[1], i, &el);
    if (napi_get_value_double(env, el, &k) != napi_ok || !(k >= 0) || k != (double)(uint64_t)k) { napi_throw_type_error(env, nullptr, "prefixLengths must be an array of non-negative integers"); return nullptr; }
    lens[i] = (uint64_t)k;
  }
  amg_buffers* l = nullptr; amg_error err;
  if (amg_get_history_patches(b, lens.data(), n, &l, &err)) return throwAmg(env, err);
  return buffersToJs(env, l);
}
// mergeMany(state, others) — src/automerge.js:61-67 at the backend level, folded over an array of backend states in one
// apply (amg_merge_many): the changes of each that `state` and the earlier ones lack, copied device to device, a change
// several hold sent once. Returns the flat patch applyChanges returns for that list. A document on another device throws an
// Error with code 'AMG_UNSUPPORTED' and changes nothing (js/index.js then applies the changes itself).
napi_value MergeMany(napi_env env, napi_callback_info info) {
  napi_value argv[2]; amg_backend* dst; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &dst)) return nullptr;
  bool isArray = false; napi_is_array(env, argv[1], &isArray);
  if (!isArray) { napi_throw_type_error(env, nullptr, "expected an array of backend states"); return nullptr; }
  uint32_t n = 0; napi_get_array_length(env, argv[1], &n);
  std::vector<amg_backend*> srcs(n);
  for (uint32_t i = 0; i < n; i++) { napi_value v; napi_get_element(env, argv[1], i, &v); if (!getBackend(env, v, &srcs[i])) return nullptr; }
  amg_patch* patch = nullptr; amg_error err;
  if (amg_merge_many(dst, srcs.data(), n, 1, &patch, &err)) {
    if (err.code == AMG_UNSUPPORTED) { napi_throw_error(env, "AMG_UNSUPPORTED", err.msg); return nullptr; }
    return throwAmg(env, err);
  }
  return patchToJs(env, patch);
}
// applyLocalChangeTable(state, table) — backend/backend.js:54-91 applyLocalChange with the change request given as a change
// table (layout: amgpu.h) holding one change: encoded with the author's previous change hash added to its deps and applied
// on the device (amg_apply_local_change). Returns [patch, change]: the flat patch without the new change's hash in its deps,
// and the binary change as encodeChange returns it.
napi_value ApplyLocalChangeTable(napi_env env, napi_callback_info info) {
  napi_value argv[2]; amg_backend* b; if (!getArgs(env, info, 2, argv) || !getBackend(env, argv[0], &b)) return nullptr;
  const uint8_t* p; size_t len; if (!getBytes(env, argv[1], &p, &len)) return nullptr;
  amg_patch* patch = nullptr; amg_buffers* change = nullptr; amg_error err;
  if (amg_apply_local_change(b, p, len, 1, &patch, &change, &err)) return throwAmg(env, err);
  napi_value out, ch; napi_create_array_with_length(env, 2, &out);
  napi_get_element(env, buffersToJs(env, change), 0, &ch);
  napi_set_element(env, out, 0, patchToJs(env, patch)); napi_set_element(env, out, 1, ch);
  return out;
}
// Backend.free — backend/backend.js:16-19: releases the device memory now instead of at garbage collection
napi_value Free(napi_env env, napi_callback_info info) {
  napi_value argv[1]; Holder* h; if (!getArgs(env, info, 1, argv) || !getHolder(env, argv[0], &h)) return nullptr;
  if (h->b) { amg_free(h->b); h->b = nullptr; }
  napi_value u; napi_get_undefined(env, &u); return u;
}

napi_value InitModule(napi_env env, napi_value exports) {
  struct { const char* name; napi_callback fn; } fns[] = {
    {"init", Init}, {"load", Load}, {"clone", Clone}, {"free", Free}, {"applyChanges", ApplyChanges}, {"getPatch", GetPatch}, {"save", Save},
    {"getHeads", GetHeads}, {"getChanges", GetChanges}, {"getChangesAdded", GetChangesAdded}, {"getChangeByHash", GetChangeByHash},
    {"getMissingDeps", GetMissingDeps}, {"clockOf", ClockOf}, {"hashByActor", HashByActor}, {"syncBloom", SyncBloom},
    {"syncChangesToSend", SyncChangesToSend}, {"decodeChanges", DecodeChanges}, {"decodeHistory", DecodeHistory},
    {"encodeChanges", EncodeChanges}, {"historyPatches", HistoryPatches}, {"mergeMany", MergeMany},
    {"applyLocalChangeTable", ApplyLocalChangeTable}};
  for (auto& f : fns) { napi_value fn; napi_create_function(env, f.name, NAPI_AUTO_LENGTH, f.fn, nullptr, &fn); napi_set_named_property(env, exports, f.name, fn); }
  return exports;
}

}  // namespace

NAPI_MODULE(NODE_GYP_MODULE_NAME, InitModule)
