// amgpu backend for automerge-classic: the module shape of backend/index.js:1-8, to be handed to
// Automerge.setDefaultBackend() (src/automerge.js:147-149) or to the reference's own test-suite through
// WASM_BACKEND_PATH (test/wasm.js:12-25). The document lives on the GPU behind the N-API addon (addon/amgpu_napi.cc ->
// include/amgpu.h); what stays in JavaScript is what the reference keeps outside BackendDoc: the frozen-handle protocol
// (backend/util.js:1-10), applyLocalChange's bookkeeping (backend/backend.js:54-91) with the reference's own encodeChange,
// and the inflation of the flat patch into the Patch object (./inflate_patch.js).
'use strict'

const native = require('../addon/build/Release/amgpu_napi')
const { encodeChange } = require('automerge/backend/columnar')   // stays JS, exactly as in backend.js:83
const { inflatePatch } = require('./inflate_patch')

const OUTDATED = 'Attempting to use an outdated Automerge document that has already been updated. ' +
  'Please use the latest document state, or call Automerge.clone() if you really need to use this old document state.'

function backendState(backend) {                                   // backend/util.js:1-10
  if (backend.frozen) throw new Error(OUTDATED)
  return backend.state
}
const toHex = bytes => Array.from(bytes, b => (b < 16 ? '0' : '') + b.toString(16)).join('')
function fromHex(list) {                                           // hashes travel as n x 32 bytes
  const out = new Uint8Array(32 * list.length)
  list.forEach((h, i) => { for (let k = 0; k < 32; k++) out[32 * i + k] = parseInt(h.substr(2 * k, 2), 16) })
  return out
}
const actorBytes = actor => { const out = new Uint8Array(actor.length / 2); for (let k = 0; k < out.length; k++) out[k] = parseInt(actor.substr(2 * k, 2), 16); return out }
const heads = state => native.getHeads(state).map(toHex)

function init() { return {state: native.init(), heads: []} }                                         // backend.js:8-10
function clone(backend) { return {state: native.clone(backendState(backend)), heads: backend.heads} } // backend.js:12-14
function free(backend) { native.free(backend.state); backend.state = null; backend.frozen = true }    // backend.js:16-19

function applyChanges(backend, changes) {                          // backend.js:27-32
  const state = backendState(backend)
  if (changes instanceof Uint8Array) throw new TypeError('applyChanges takes an array of Uint8Arrays, not just a single Uint8Array')
  const patch = inflatePatch(native.applyChanges(state, changes, false, true), false)
  backend.frozen = true
  return [{state, heads: patch.deps}, patch]
}

function hashByActor(state, actorId, index) {                      // backend.js:34-45
  const h = native.hashByActor(state, actorBytes(actorId), index)
  if (h) return toHex(h)
  throw new RangeError(`Unknown change: actorId = ${actorId}, seq = ${index + 1}`)
}

function applyLocalChange(backend, change) {                       // backend.js:54-91, unchanged logic
  const state = backendState(backend)
  if (change.seq <= native.clockOf(state, actorBytes(change.actor))) throw new RangeError('Change request has already been applied')
  if (change.seq > 1) {                                            // the local actor's previous change is an implicit dependency
    const lastHash = hashByActor(state, change.actor, change.seq - 2)
    const deps = {[lastHash]: true}
    for (const h of change.deps) deps[h] = true
    change.deps = Object.keys(deps).sort()
  }
  const binaryChange = encodeChange(change)
  const patch = inflatePatch(native.applyChanges(state, [binaryChange], true, true), false)   // isLocal: patch carries actor and seq (new.js:1874-1877)
  backend.frozen = true
  const lastHash = hashByActor(state, change.actor, change.seq - 1)
  patch.deps = patch.deps.filter(head => head !== lastHash)        // the change itself is not a dependency of the next one
  return [{state, heads: heads(state)}, patch, binaryChange]
}

function save(backend) { return native.save(backendState(backend)) }                                   // backend.js:93-95
function load(data) { const state = native.load(data); return {state, heads: heads(state)} }           // backend.js:104-107
function loadChanges(backend, changes) {                           // backend.js:116-121
  const state = backendState(backend)
  native.applyChanges(state, changes, false, false)
  backend.frozen = true
  return {state, heads: heads(state)}
}
function getPatch(backend) { return inflatePatch(native.getPatch(backendState(backend)), true) }       // backend.js:127-129
function getHeads(backend) { return backend.heads }                                                    // backend.js:135-137
function getAllChanges(backend) { return getChanges(backend, []) }                                     // backend.js:142-144
function getChanges(backend, haveDeps) {                           // backend.js:151-156
  if (!Array.isArray(haveDeps)) throw new TypeError('Pass an array of hashes to Backend.getChanges()')
  return native.getChanges(backendState(backend), fromHex(haveDeps))
}
function getChangesAdded(backend1, backend2) { return native.getChangesAdded(backendState(backend1), backendState(backend2)) }   // backend.js:166-168
function getChangeByHash(backend, hash) { return native.getChangeByHash(backendState(backend), fromHex([hash])) }               // backend.js:176-178
function getMissingDeps(backend, heads = []) { return native.getMissingDeps(backendState(backend), fromHex(heads)).map(toHex) } // backend.js:190-192
// getHistory's snapshots (src/automerge.js:105-118): for every k, the patch getPatch(loadChanges(init(), getAllChanges(backend).slice(0, k)))
// returns, filtered on the device from the document's op table; no change is re-sent
function historyPatches(backend, prefixLengths) {
  return native.historyPatches(backendState(backend), prefixLengths).map(flat => inflatePatch(flat, true))
}

// Automerge.merge (src/automerge.js:61-67) at the backend level: applyChanges(backend1, getChangesAdded(backend1, backend2)),
// with the changes copied from backend2's device memory to backend1's. backend1 is frozen, as applyChanges freezes it.
// Documents on different devices take the same route through JavaScript.
function merge(backend1, backend2) {
  const state = backendState(backend1), other = backendState(backend2)
  let flat
  try { flat = native.merge(state, other) } catch (e) {
    if (e.code !== 'AMG_UNSUPPORTED') throw e
    return applyChanges(backend1, getChangesAdded(backend1, backend2))
  }
  const patch = inflatePatch(flat, false)
  backend1.frozen = true
  return [{state, heads: patch.deps}, patch]
}

const backendApi = { init, clone, free, applyChanges, applyLocalChange, save, load, loadChanges, getPatch,
  getHeads, getAllChanges, getChanges, getChangesAdded, getChangeByHash, getMissingDeps, historyPatches, merge }

// backend/sync.js:19 hard-imports './backend': the sync functions of backend/index.js are re-created over this backend by
// loading the reference's sync.js with its backend import redirected (it only calls getHeads / getChanges /
// getChangeByHash / getMissingDeps / applyChanges).
function bindSync() {
  const Module = require('module'), path = require('path')
  const syncPath = require.resolve('automerge/backend/sync'), backendPath = path.join(path.dirname(syncPath), 'backend.js')
  const saved = require.cache[backendPath]
  require.cache[backendPath] = Object.assign(new Module(backendPath), {exports: backendApi, loaded: true, filename: backendPath})
  delete require.cache[syncPath]
  const sync = require(syncPath)
  if (saved) require.cache[backendPath] = saved; else delete require.cache[backendPath]
  return sync
}
let sync = null
for (const name of ['generateSyncMessage', 'receiveSyncMessage', 'encodeSyncMessage', 'decodeSyncMessage', 'initSyncState', 'encodeSyncState', 'decodeSyncState']) {
  backendApi[name] = (...args) => { if (!sync) sync = bindSync(); return sync[name](...args) }
}

module.exports = backendApi
