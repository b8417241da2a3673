"""amgpu — H100-native bulk change-replay engine behind automerge-classic's Backend API.

    from automerge_classic_b200 import Backend          # init / applyChanges / getPatch / ... (backend/index.js:1-8)

The module object `Backend` mirrors the module a caller hands to `Automerge.setDefaultBackend()`.
"""
from .backend import Backend as _Facade, backend_state as _backend_state
from .engine import GpuBackendDoc, AmgError, Unsupported, FlatChanges, decode_changes as _decode_changes, _decoder_for

from . import sync as _sync


def bind_sync(facade, device=True):
    """Adds the sync functions of backend/index.js:2, 7 to a Backend facade (the reference's sync.js is tied to its own backend).
    device=False keeps the Bloom filters and the choice of changes to send in Python (see sync.Sync)."""
    s = _sync.Sync(facade, device=device)
    facade.generateSyncMessage, facade.receiveSyncMessage = s.generateSyncMessage, s.receiveSyncMessage
    for name in ('encodeSyncMessage', 'decodeSyncMessage', 'encodeSyncState', 'decodeSyncState', 'initSyncState'):
        setattr(facade, name, getattr(_sync, name))
    return facade


def decodeChanges(binary_changes):
    """Automerge.decodeChanges (columnar.js:843-857) on the device: a list of change objects."""
    return _decode_changes(binary_changes)


def decodeChange(buf):
    """Automerge.decodeChange (columnar.js:770-776, src/automerge.js:154): one binary change -> its change object."""
    return _decoder_for(GpuBackendDoc).decode_changes_flat([buf]).to_changes()[0]


def encodeChanges(changes):
    """Automerge.encodeChange over a list of change objects, in one device call: their binary changes."""
    return _decoder_for(GpuBackendDoc).encode_flat(FlatChanges.from_changes(changes))[0]


def encodeChange(change):
    """Automerge.encodeChange (columnar.js:710-739, src/automerge.js:153): a change object -> its binary change. A `hash` that
    differs from the encoding's raises the reference's RangeError (columnar.js:735-737)."""
    out, hashes = _decoder_for(GpuBackendDoc).encode_flat(FlatChanges.from_changes([change]))
    if change.get('hash') and change['hash'] != hashes[0]:
        raise AmgError(1, 'Change hash does not match encoding: %s != %s' % (change['hash'], hashes[0]))
    return out[0]


class HistoryEntry:
    """One entry of getHistory: `change` and `snapshot` are computed when first read, like the reference's getters."""

    def __init__(self, history, index):
        self._history, self._index = history, index

    @property
    def change(self):
        """decodeChange of the entry's change (all of the list's changes are decoded in one device call, once)."""
        h = self._history
        if h['changes'] is None:
            h['changes'] = h['doc'].decode_history_flat().to_changes()
        return h['changes'][self._index]

    @property
    def snapshot(self):
        """The patch getPatch(loadChanges(init(), history[:index + 1])) returns, filtered on the device from the document's op
        table. There is no frontend here, so it is the patch, not a document."""
        return self._history['doc'].history_patches([self._index + 1])[0]


def getHistory(backend):
    """Automerge.getHistory (src/automerge.js:105-118) at the backend level: one entry per change of getAllChanges(backend).
    No change bytes leave the device. Later changes to the document only append to getAllChanges order, so the entries
    stay valid."""
    doc = _backend_state(backend)
    n = sum(doc.clock().values())   # every actor's changes have seq 1 .. clock[actor]
    history = {'doc': doc, 'changes': None}
    return [HistoryEntry(history, i) for i in range(n)]


def merge(local, remote):
    """Automerge.merge (src/automerge.js:61-67) at the backend level: [newLocalHandle, patch], where the patch is the one
    applyChanges(local, getChangesAdded(local, remote)) returns. The changes go from remote's device memory to local's
    without leaving the device. The local handle is frozen, as applyChanges freezes it; remote is not changed. When the
    document class has no device merge, or the engine declines (Unsupported, e.g. documents on different devices), the
    changes take the host route."""
    state, other = _backend_state(local), _backend_state(remote)
    patch = None
    if hasattr(state, 'merge'):
        try:
            patch = state.merge(other)
        except Unsupported:
            pass   # nothing changed: the host route below
    if patch is None:
        patch = state.apply_changes(other.get_changes_added(state))
    local['frozen'] = True
    return [{'state': state, 'heads': state.heads()}, patch]


Backend = bind_sync(_Facade(GpuBackendDoc))
__all__ = ['Backend', 'GpuBackendDoc', 'AmgError', 'Unsupported', 'bind_sync', 'decodeChange', 'decodeChanges', 'encodeChange', 'encodeChanges',
           'getHistory', 'HistoryEntry', 'merge']
