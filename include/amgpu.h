/* amgpu — C ABI of the H100-native bulk change-replay engine for automerge-classic.
 *
 * This is the drop-in boundary: a backend module for `Automerge.setDefaultBackend()`
 * (reference src/automerge.js:147-149; function set in backend/index.js:1-8 and
 * @types/automerge/index.d.ts:139-162) binds exactly these entry points through N-API (see
 * INTEGRATION.md for the shim); the Python mirror in automerge_classic_b200/engine.py binds them
 * through ctypes. Plain pointers and sizes only. Every call is synchronous (the reference backend is
 * synchronous: backend/backend.js:27-32). There is no CPU fallback: amg_init fails when no CUDA
 * device is present.
 *
 * Error convention (reference: synchronous `throw` of RangeError / TypeError, state unchanged,
 * backend/new.js:1793-1795): functions return 0 on success, otherwise an amg_error_code, and fill
 * `err->msg` with the reference's message text (e.g. "no matching operation for pred: 3@abcd").
 */
#ifndef AMGPU_H
#define AMGPU_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct amg_backend amg_backend;   /* one document: replaces class BackendDoc, backend/new.js:1694 */
typedef struct amg_patch amg_patch;       /* flat binary patch, see "patch layout" below */
typedef struct amg_buffers amg_buffers;   /* a list of byte buffers returned by the library */

typedef enum { AMG_OK = 0, AMG_RANGE_ERROR = 1, AMG_TYPE_ERROR = 2, AMG_INTERNAL_ERROR = 3, AMG_UNSUPPORTED = 4, AMG_CUDA_ERROR = 5 } amg_error_code;
typedef struct { int code; char msg[512]; } amg_error;

/* Backend.init()  — backend/backend.js:8-10 (new BackendDoc(), new.js:1751-1767) */
amg_backend* amg_init(int cuda_device, amg_error* err);
/* Backend.clone() — backend/backend.js:12-14 (BackendDoc.clone, new.js:1773-1790) */
amg_backend* amg_clone(amg_backend* b, amg_error* err);
/* Backend.load(data) — backend/backend.js:104-107 -> new BackendDoc(buffer), new.js:1709-1750 (document chunk, type 0) */
amg_backend* amg_load(int cuda_device, const uint8_t* data, size_t len, amg_error* err);
/* Backend.free()  — backend/backend.js:16-19 */
void amg_free(amg_backend* b);

/* Drops the document but keeps every device / pinned allocation (steady-state serving, benchmarking). */
int amg_reset(amg_backend* b, amg_error* err);
/* Pre-sizes the change arena (pinned host mirror + device) so that a bulk replay does not grow it mid-call. */
int amg_reserve(amg_backend* b, size_t arena_bytes, amg_error* err);

/* Backend.applyChanges(state, changes) — backend/backend.js:27-32 -> BackendDoc.applyChanges, new.js:1797-1879.
 * `bufs[i]` / `lens[i]`: the binary changes (chunk type 1, or 2 = DEFLATE, inflated on the device by an RFC 1951 decoder,
 * csrc/inflate.cuh, where columnar.js:813-823 uses pako). is_local != 0 mirrors the `isLocal` argument used by applyLocalChange
 * (backend.js:84): the patch then carries actor and seq of the single change. want_patch == 0 is
 * Backend.loadChanges (backend.js:116-121): same state transition, no patch computed; *out is set to NULL. */
int amg_apply_changes(amg_backend* b, const uint8_t* const* bufs, const size_t* lens, size_t n, int is_local, int want_patch,
                      amg_patch** out, amg_error* err);
/* Same, with the n changes stored back to back in one buffer: change i is blob[offsets[i] .. offsets[i+1]) (offsets: host
 * memory). This is the bulk-replay entry point. `blob` may be pinned host memory (uploaded in 16 MB pieces, each piece
 * hashed and decoded while the next one is in flight), pageable host memory (staged through the engine's pinned arena
 * mirror) or DEVICE memory (copied device to device: the bytes are already resident). */
int amg_apply_changes_packed(amg_backend* b, const uint8_t* blob, const uint64_t* offsets, size_t n, int is_local, int want_patch,
                             amg_patch** out, amg_error* err);
/* Backend.getPatch(state) — backend/backend.js:127-129 -> new.js:2060-2068 / documentPatch new.js:1604-1635 */
int amg_get_patch(amg_backend* b, amg_patch** out, amg_error* err);

/* header-only patch: maxOp, clock, deps (heads), pendingChanges and the actor table, without diffs */
int amg_get_state(amg_backend* b, amg_patch** out, amg_error* err);

/* Backend.getHeads — backend.js:135-137: n hashes of 32 bytes, ascending */
/* Backend.save (backend/backend.js:93-95, new.js:2033-2055): one buffer = the document chunk */
int amg_save(amg_backend* b, amg_buffers** out, amg_error* err);
int amg_get_heads(amg_backend* b, amg_buffers** out, amg_error* err);
/* Backend.getAllChanges / getChanges(haveDeps) — backend.js:142-156 -> new.js:1921-1973; have_deps = n hashes x 32 bytes.
 * The reference's traversal runs on the host over a graph of change indexes the engine keeps: dependencies resolved on the
 * device (by the causal gate of applyChanges, or from the change headers for loaded changes), brought up to date by each
 * query, with the changes' hashes, against which have_deps are looked up. */
int amg_get_changes(amg_backend* b, const uint8_t* have_deps, size_t n, amg_buffers** out, amg_error* err);
/* Backend.getChangesAdded(old, new) — backend.js:166-168 -> new.js:1979-1997. The changes of b_new that b_old lacks are
 * found by hash lookups on the device and ordered on the host over their dependency indexes; no host hash graph is built.
 * A loaded document's history is rebuilt first (both documents). The two documents must be on the same CUDA device
 * (AMG_UNSUPPORTED otherwise). */
int amg_get_changes_added(amg_backend* b_new, amg_backend* b_old, amg_buffers** out, amg_error* err);
/* Automerge.merge(localDoc, remoteDoc) — src/automerge.js:61-67, at the backend level: applyChanges(dst, getChangesAdded(dst,
 * src)) (backend.js:27-32, 166-168) without the changes leaving the device. The changes of src that dst lacks, in
 * getChangesAdded's order, are copied from src's arena into one device buffer and applied to dst through the device-memory
 * path of amg_apply_changes_packed; *out is the patch that applyChanges returns (want_patch == 0: none, *out = NULL).
 *   - No changes to send (src == dst, src a clone of dst, src's changes a subset of dst's): dst applies an empty batch and
 *     *out is the patch applyChanges(dst, []) returns (queued changes of dst are retried, as always).
 *   - src's queued changes are never sent; dst's queued changes may become applicable.
 *   - src is not changed (a loaded src has its history rebuilt first, as getChangesAdded does; so has a loaded dst).
 *   - A change getChangesAdded would hand over DEFLATEd because the engine rebuilt it (>= 256 bytes) goes over in plain
 *     form; dst returns it DEFLATEd from getChanges, getChangeByHash, getChangesAdded and sync, as it would after the host
 *     route. Only amg_arena shows the plain bytes.
 *   - dst and src on different CUDA devices: AMG_UNSUPPORTED, nothing changed (amg_get_changes_added declines them too).
 *   - An apply error (e.g. both documents hold a different change for the same actor and seq) is the error applyChanges
 *     reports for the same changes, and dst is unchanged. */
int amg_merge(amg_backend* dst, amg_backend* src, int want_patch, amg_patch** out, amg_error* err);
/* device span of the last amg_merge call in ms, lookups, copy and apply (CUDA events on dst's main stream, like amg_last_history_ms) */
float amg_last_merge_ms(amg_backend* dst);
/* Backend.getChangeByHash — backend.js:176-178 -> new.js:1999-2002; zero buffers when unknown */
int amg_get_change_by_hash(amg_backend* b, const uint8_t hash[32], amg_buffers** out, amg_error* err);
/* Backend.getMissingDeps — backend.js:190-192 -> new.js:2014-2028: hashes of 32 bytes, ascending. The queued changes are
 * hashed and parsed on the device; their dependencies and `heads` are looked up among the applied and queued hashes there. */
int amg_get_missing_deps(amg_backend* b, const uint8_t* heads, size_t n, amg_buffers** out, amg_error* err);
/* backend/backend.js:54-91 applyLocalChange. `table`: a change table (amg_decode_changes layout) holding one change request;
 * pinned, pageable or device memory. *out: the patch applyChanges(isLocal) returns, without the new change's hash in its deps
 * (want_patch == 0: none). *out_change: one buffer, the binary change as encodeChange returns it.
 *   - The author is actor entry 0 of the change. seq <= clock[author]: AMG_RANGE_ERROR "Change request has already been
 *     applied"; seq - 1 > clock[author]: AMG_RANGE_ERROR "Unknown change: actorId = <hex>, seq = <seq - 1>".
 *   - For seq > 1 the hash of the author's change seq - 1 is added to the deps; the deps are then sorted and without
 *     repeats (backend.js:76-79). It is read from the engine's hashes on the device; no host hash graph is built. A loaded
 *     document has its history rebuilt first unless that change is one of the loaded heads.
 *   - The change is encoded and applied on the device; its bytes go to the host only after the apply. Encoder errors
 *     are those of amg_encode_changes, apply errors those of amg_apply_changes. A table that does not hold exactly one
 *     change is AMG_RANGE_ERROR.
 *   - On every error above the document is unchanged. The exception is a change whose deps are not all applied: it waits
 *     in the queue, and the call then fails with "Unknown change: ..., seq = <seq>", as the reference does after its apply.
 *   - A change of 256 bytes or more is returned DEFLATEd, and getChanges, getChangeByHash, getChangesAdded and sync hand it
 *     out DEFLATEd, byte for byte as after applying the DEFLATEd form. Only amg_arena shows the plain bytes. */
int amg_apply_local_change(amg_backend* b, const uint8_t* table, size_t table_len, int want_patch,
                           amg_patch** out, amg_buffers** out_change, amg_error* err);
/* device span of the last amg_apply_local_change call in ms: staging, encode, apply and the read-back of the change */
float amg_last_local_ms(amg_backend* b);
/* state needed by the host-side applyLocalChange (backend.js:54-91): clock[actor] and hashesByActor[actor][index] */
int amg_clock_of(amg_backend* b, const uint8_t* actor, size_t actor_len, uint64_t* seq_out, amg_error* err);
int amg_hash_by_actor(amg_backend* b, const uint8_t* actor, size_t actor_len, uint64_t index, uint8_t hash_out[32], int* found, amg_error* err);

/* sync.js:234-238 makeBloomFilter: the Bloom filter (BloomFilter(...).bytes, sync.js:38-76) over the hashes of
 * getChanges(b, last_sync); last_sync = n hashes x 32 bytes. One buffer; empty when there are no such changes. The probes
 * are set on the device from the hashes the engine holds; n == 0 (every change) does not build the host hash graph.
 * An unknown hash fails like amg_get_changes ("hash not found"). */
int amg_sync_bloom(amg_backend* b, const uint8_t* last_sync, size_t n, amg_buffers** out, amg_error* err);
/* sync.js:246-306 getChangesToSend for have.length > 0. last_sync: the union of have[i].lastSync in first-seen order
 * (n_last x 32 bytes); filters: n_filters already-parsed peer Bloom filters {num_entries, num_probes, bits, bits_len};
 * need: n_need x 32 bytes. out_changes: the changes to send, in the reference's order; out_hashes: one buffer of
 * 32-byte hashes back to back, one per returned change (the caller filters sentHashes with them). A filter with more than 64 probes
 * fails with AMG_UNSUPPORTED (the caller answers from its host implementation instead). */
typedef struct { uint32_t num_entries, num_probes; const uint8_t* bits; size_t bits_len; } amg_bloom;
int amg_sync_changes_to_send(amg_backend* b, const uint8_t* last_sync, size_t n_last, const amg_bloom* filters, size_t n_filters,
                             const uint8_t* need, size_t n_need, amg_buffers** out_changes, amg_buffers** out_hashes, amg_error* err);

/* columnar.js:770-776 decodeChange over n change containers (chunk type 1 or 2, one per entry, as in amg_apply_changes_packed:
 * change i is blob[offsets[i] .. offsets[i+1]); blob may be pinned, pageable or device memory). The bytes are staged into
 * scratch, DEFLATEd changes inflated on the device; the document is not touched. One buffer: the change table (layout below).
 * On error, *failed_index is the change the reference's sequential loop fails on first, and err carries its message. */
int amg_decode_changes(amg_backend* b, const uint8_t* blob, const uint64_t* offsets, size_t n,
                       amg_buffers** out, size_t* failed_index, amg_error* err);
/* the same for every applied change of b, in getAllChanges order (new.js:1925-1927), read in place from device memory (a
 * loaded document's history is rebuilt first, as getChanges does). Queued changes are not included. */
int amg_decode_history(amg_backend* b, amg_buffers** out, amg_error* err);
/* device span of the last amg_decode_changes / amg_decode_history call in ms (CUDA events on the engine's main stream) */
float amg_last_decode_ms(amg_backend* b);
/* Change table layout (little endian). A header of 12 uint64:
 *   [0] 0x31474843474d41 ("AMGCHG1") [1] nChanges [2] changesOff [3] nOps [4] opsOff [5] nPreds [6] predsOff
 *   [7] nActors [8] actorsOff [9] bytesOff [10] bytesLen [11] 0
 * followed by the sections (offsets relative to the start of the buffer):
 *   changes: nChanges x { uint8 hash[32]; uint64 seq, startOp; int64 time; uint32 msgOff, msgLen, depsOff, nDeps, actorFirst,
 *            nActors, extraOff, extraLen, hasExtra, pad; uint64 firstOp, nOps, firstPred, nPreds }          (128 bytes)
 *   ops    : nOps x { uint32 objActor, objCtr, keyActor, keyCtr, keyStrOff, keyStrLen, insert, action, valLen, valOff,
 *            chldActor, chldCtr, predFirst, predNum, change, pad }                                             (64 bytes)
 *   preds  : nPreds x { uint32 actor, ctr }
 *   actors : nActors x { uint32 off, len }: per change, entries actorFirst .. actorFirst + nActors - 1 are its actor table
 *            (entry 0 is the author); the op and pred actor numbers index it
 *   bytes  : the decoded change containers back to back (inflated)
 * 0xffffffff is null (keyStrLen null: no key string column value; an empty string has length 0). msgOff, depsOff (nDeps x 32
 * bytes), extraOff, keyStrOff, valOff and the actor entries' off are offsets INTO THE TABLE. action is the raw action number,
 * valLen the VALUE_LEN tag (length << 4 | type, columnar.js:46-49); every value has been checked like decodeValue does.
 *
 * What amg_encode_changes reads of a table: the header's changes, ops, preds and actors sections; per change seq, startOp,
 * time, the message, the deps (hashes, any order), the extra bytes when hasExtra is set, actorFirst / nActors and firstOp /
 * nOps; per op every field but `change` and `pad`; preds (any order). It ignores the hash, the bytes section (bytesOff /
 * bytesLen: the offsets point anywhere into the table), pad and the change's firstPred / nPreds beyond a range check (the ops'
 * predFirst / predNum say which preds are theirs). A change's actor table is only the mapping from its actor numbers to
 * actor ids: the encoder writes the canonical one (author first, then the actors the ops use, sorted by id bytes), so
 * unused, repeated or unsorted entries encode like the canonical table. keyStrLen > 0 is a map key; otherwise keyCtr 0 with
 * insert is _head and keyCtr > 0 an element id. A value is written for action 1 (set) and 5 (inc) only. */
/* columnar.js:710-739 encodeChange over the n changes of a change table in the layout amg_decode_changes returns (table may
 * be pinned, pageable or device memory; table_len bytes). out_changes: n binary changes as encodeChange returns them, i.e.
 * chunk type 2 (zlib level 6, columnar.js:738, 798-808) when the plain change is >= 256 bytes; out_hashes: one buffer of
 * n x 32 bytes. On error *failed_index is the smallest failing change (a damaged table is AMG_RANGE_ERROR naming the change;
 * a damaged header names change 0). A change whose encoding may reach 4 GiB (its ops may share one value or key
 * string) is AMG_UNSUPPORTED, found before anything is sized. The document is not touched. */
int amg_encode_changes(amg_backend* b, const uint8_t* table, size_t table_len, amg_buffers** out_changes,
                       amg_buffers** out_hashes, size_t* failed_index, amg_error* err);
/* device span of the last amg_encode_changes call in ms (CUDA events on the engine's main stream, like amg_last_decode_ms) */
float amg_last_encode_ms(amg_backend* b);

/* src/automerge.js:105-118 getHistory: the `snapshot` of history entry k - 1 is built from the first k changes of
 * getAllChanges order (application order; for a loaded document its stored changes first): Frontend.applyPatch(init(),
 * backend.getPatch(backend.loadChanges(backend.init(), history.slice(0, k)))). This returns that getPatch for every
 * k = prefix_lens[i]: n self-contained flat patches in the amg_patch_bytes layout, one buffer per length in the order given
 * (lengths may repeat and need not be sorted). Such a prefix is causally closed, so each patch is computed from the
 * document's own op table, filtered to the ops of the prefix's changes, without re-sending any change: pendingChanges is 0,
 * deps are the prefix's heads, clock and maxOp its own; the actor table is the document's (its clock lists only the
 * prefix's actors). k = 0 gives the patch of getPatch(init()). Queued changes are never part of a prefix. A length greater
 * than the number of applied changes is AMG_RANGE_ERROR. A loaded document's history is rebuilt first, as amg_get_changes
 * does (AMG_UNSUPPORTED for a loaded document that holds columns with unknown ids). The document is not touched. */
int amg_get_history_patches(amg_backend* b, const uint64_t* prefix_lens, size_t n, amg_buffers** out, amg_error* err);
/* device span of the last amg_get_history_patches call in ms (CUDA events on the engine's main stream, like amg_last_decode_ms) */
float amg_last_history_ms(amg_backend* b);

/* returned buffer lists */
size_t amg_buffers_count(const amg_buffers* l);
const uint8_t* amg_buffers_get(const amg_buffers* l, size_t i, size_t* len);
void amg_buffers_free(amg_buffers* l);

/* Patch layout (little endian). amg_patch_bytes returns a header of 20 uint64:
 *   [0] 0x31504747414d41 ("AMAGGP1") [1] maxOp [2] pendingChanges [3] hasActorSeq [4] seq [5] actorOff [6] actorLen
 *   [7] actorsOff [8] nActors [9] clockOff [10] nClock [11] depsOff [12] nDeps [13] propsOff [14] nProps
 *   [15] editsOff [16] nEdits [17] editElemOff [18] bytesOff [19] bytesLen
 * followed by the sections (offsets relative to the start of the buffer, 8-byte aligned):
 *   actors : nActors x { uint32 len; bytes[len]; pad to 4 }   (document actor index -> actor id bytes)
 *   clock  : nClock x { uint64 actorIndex; uint64 seq }
 *   deps   : nDeps x 32 bytes
 *   props  : nProps x { uint64 objId; uint64 opId; uint32 keyOff, keyLen, valLen, valOff, flags, pad }   (map entries)
 *   edits  : nEdits x { uint64 objId; uint64 opId; uint32 index, kind, valLen, valOff }                  (list edits, per object in order)
 *   editElem: nEdits x uint64 elemId (offset 0 in the header = section absent: every insert's elemId is its opId)
 *   bytes  : the map keys and value payloads the records refer to, gathered on the device
 * ids are (counter << 16 | actorIndex); objId 0 = _root. keyOff / valOff are offsets INTO THE PATCH BUFFER (its bytes
 * section): a patch is self-contained, no second buffer is needed to read it. valLen is the reference's VALUE_LEN tag
 * (length << 4 | type, columnar.js:46-49); numeric payloads have been validated like the reference's decodeValue does
 * (columnar.js:300-329) - a malformed one makes the call fail with the reference's RangeError.
 * props.flags = action << 8 | 1 if the key has no visible value (reference emits `key: {}`);
 * edits.kind = (0 insert | 1 remove | 2 update) | 0x100 if the edit starts a new run (edits without the bit
 * continue the previous insert as `multi-insert` / add to the previous remove's count, new.js:747-782)
 * | 0x1000 for a counter whose increments were summed: its value is the int64 (valOff << 32 | valLen)
 * | 0x200 if the insert is rendered as `multi-insert` (set on every member of a run, and on a run start whose
 * followers were popped again by appendUpdate, new.js:811-813) | action << 16.
 * The nested Patch object of @types/automerge/index.d.ts:236-316 is assembled from this by the binding. */
/* The bytes live in a pinned buffer owned by the backend: valid until the next call on the same backend. */
const uint8_t* amg_patch_bytes(const amg_patch* p, size_t* len);
void amg_patch_free(amg_patch* p);
/* host copy of the document arena (every change's bytes back to back, inflated copies of DEFLATEd changes behind them);
 * valid until the next mutating call. The engine keeps no host copy of bytes that were handed over in pinned or device
 * memory: the missing part is fetched from the device by this call (and by getChanges & co, which read from it). */
const uint8_t* amg_arena(amg_backend* b, size_t* len);

/* ---- parity / measurement hooks (not part of the reference surface) ---- */
/* decoded rows of a batch of changes (SoA dump of the decode kernels' output, gathered into batch order), for parity tests
 * (SURVEY.md 8c "parity definition" items 1-2: per-change hash, decoded rows). rows_out (malloc'ed, amg_free_mem) holds 12
 * columns x total_ops {objActor,objCtr,keyActor,keyCtr,keyStrOff,keyStrLen,insert,action,valLen,valOff,predNum,predOff}
 * (change-local actor indexes, 0xffffffff = null, offsets relative to the staged copy of the batch) followed by
 * 2 columns x total_preds {predActor, predCtr}. The document is not touched. */
int amg_debug_decode(amg_backend* b, const uint8_t* blob, const uint64_t* offsets, size_t n, uint8_t* hashes_out /* n*32 */,
                     uint32_t* n_ops_out /* n */, uint32_t** rows_out, size_t* total_ops, size_t* total_preds, amg_error* err);
/* document-ordered op table: rows[n][8] = {objCtr,objActor,idCtr,idActor,keyCtr,keyActor,flags,succNum}; succ[m][2] = {ctr, actor} */
int amg_debug_dump_ops(amg_backend* b, uint64_t** rows_out, size_t* n, uint64_t** succ_out, size_t* m, amg_error* err);
/* timings of the last applyChanges call: [0..11] CUDA-event phases in ms on the engine's main stream (upload + hash + decode of
 * the pieces, inflate + rest of the decode, gate, actors + seq + row finalisation, op set, patch groups + props, list index,
 * edits + copy-out, heads + commit), [12..23] host wall-clock marks (ms since the call started; [23] = the whole ABI call) */
int amg_last_timings(amg_backend* b, float* ms_out, int n);
/* device span of the last amg_sync_bloom / amg_sync_changes_to_send call in ms: CUDA events around its uploads, kernels and
 * read-backs on the engine's main stream (host work in between included when the stream waits for it) */
float amg_last_sync_ms(amg_backend* b);
/* device span of the last amg_get_changes / amg_get_change_by_hash / amg_get_missing_deps / amg_hash_by_actor call in ms
 * (CUDA events on the engine's main stream, like amg_last_sync_ms): the graph update, hashing and lookups of the query; the
 * host walks of getChanges and the copy of the returned changes are not in it */
float amg_last_graph_ms(amg_backend* b);
uint64_t amg_kernel_launches(amg_backend* b);
/* labelled host wall-clock marks of the last applyChanges call ("label=ms ..."), development aid */
size_t amg_debug_marks(amg_backend* b, char* buf, size_t cap);
void amg_free_mem(void* p);
/* one column of a document through either decoder of the load path: kind 0 = RLE of unsigned numbers, 1 = RLE of signed
 * numbers, 2 = delta column, 3 = boolean column; out[n] (INT64_MIN = null). parallel = 1: the token / record decoder for
 * long columns (returns 1 without touching out when it declines the stream); parallel = 0: the serial walker (malformed
 * input is an error, as in the reference). For differential tests of the two. */
int amg_debug_decode_column(amg_backend* b, const uint8_t* bytes, size_t len, int kind, size_t n, int parallel, int64_t* out, amg_error* err);
/* device-only re-run of the decode kernels over the last batch (inputs resident in HBM), for the roofline measurement:
 * ms_sha = SHA-256 kernel, ms_parse = fused decode (k_decode_tiles + k_decode_direct), ms_decode = DecodeColumnKernel over
 * changes of more than 16 ops (0 if none); algo_bytes = SURVEY.md 8d: encoded bytes + 48 B/op + 8 B/pred + 96 B/change */
int amg_bench_decode(amg_backend* b, int iters, float* ms_sha, float* ms_parse, float* ms_decode, uint64_t* algo_bytes, amg_error* err);

#ifdef __cplusplus
}
#endif
#endif
