"""Host-side mirror of the reference's Backend facade (backend/backend.js, backend/util.js).

Same function names, argument meaning and error behaviour as the module a caller passes to
`Automerge.setDefaultBackend()` (src/automerge.js:147-149; signatures in
@types/automerge/index.d.ts:139-162), so that parity tests read like the reference's own
test/backend_test.js.  The facade is generic over the document engine: `Backend(doc_class)` where
`doc_class` provides the BackendDoc surface (backend/new.js:1694-2069) — the product passes
`automerge_classic_b200.engine.GpuBackendDoc` (CUDA through the C ABI); tests also instantiate it
over the CPU oracle to replay the golden fixtures.

Handles are `{'state': doc, 'heads': [...], 'frozen': bool}` dicts exactly like the reference's
`{state, heads, frozen}` objects (backend/backend.js:9, 27-32; backend/util.js:1-10).
"""
from .columnar import encode_change
from .engine import AmgError, Unsupported


class RangeError(Exception):
    pass


OUTDATED = ('Attempting to use an outdated Automerge document that has already been updated. '
            'Please use the latest document state, or call Automerge.clone() if you really '
            'need to use this old document state.')


def backend_state(backend):
    """backend/util.js:1-10"""
    if backend.get('frozen'):
        raise RuntimeError(OUTDATED)
    return backend['state']


class Backend:
    def __init__(self, doc_class):
        self.doc_class = doc_class

    # backend.js:8-10
    def init(self):
        return {'state': self.doc_class(), 'heads': []}

    # backend.js:12-14
    def clone(self, backend):
        return {'state': backend_state(backend).clone(), 'heads': backend['heads']}

    # backend.js:16-19
    def free(self, backend):
        backend['state'] = None
        backend['frozen'] = True

    # backend.js:27-32
    def applyChanges(self, backend, changes):
        state = backend_state(backend)
        if isinstance(changes, (bytes, bytearray)):
            raise TypeError('applyChanges takes an array of Uint8Arrays, not just a single Uint8Array')
        if not isinstance(changes, (list, tuple)):
            raise TypeError('applyChanges takes an array of Uint8Arrays')
        patch = state.apply_changes(list(changes))
        backend['frozen'] = True
        return [{'state': state, 'heads': state.heads()}, patch]

    # backend.js:34-45
    def _hash_by_actor(self, state, actor_id, index):
        h = state.hash_by_actor(actor_id, index)
        if h:
            return h
        raise RangeError('Unknown change: actorId = %s, seq = %d' % (actor_id, index + 1))

    # backend.js:54-91. A document class with apply_local_change encodes and applies the change on the device; the checks
    # that come before the encoder in the reference run here first, from the clock, so that their errors win. The host
    # route below remains for other document classes and for a request the engine declines (Unsupported).
    def applyLocalChange(self, backend, change):
        state = backend_state(backend)
        local = getattr(state, 'apply_local_change', None)
        clock = state.clock_of(change['actor']) if local else state.clock().get(change['actor'], 0)
        if change['seq'] <= clock:
            raise RangeError('Change request has already been applied')
        if local:
            if change['seq'] - 1 > clock:
                raise RangeError('Unknown change: actorId = %s, seq = %d' % (change['actor'], change['seq'] - 1))
            try:
                patch, binary_change = local(change)
            except Unsupported:
                pass   # nothing changed: the host route
            except AmgError as e:
                # The seq checks above ran already, so "Unknown change" here means the change was applied to the queue
                # (its deps are not all applied) and has no hash yet. The reference raises this after its apply too
                # (backend.js:84-85), with the handle frozen.
                if not str(e).startswith('Unknown change: '):
                    raise
                backend['frozen'] = True
                raise RangeError(str(e)) from None
            else:
                backend['frozen'] = True
                return [{'state': state, 'heads': state.heads()}, patch, binary_change]
        change = dict(change)
        if change['seq'] > 1:
            last_hash = self._hash_by_actor(state, change['actor'], change['seq'] - 2)
            deps = {last_hash: True}
            for h in change['deps']:
                deps[h] = True
            change['deps'] = sorted(deps.keys())
        binary_change = encode_change(change)
        patch = state.apply_changes([binary_change], is_local=True)
        backend['frozen'] = True
        last_hash = self._hash_by_actor(state, change['actor'], change['seq'] - 1)
        patch['deps'] = [h for h in patch['deps'] if h != last_hash]
        return [{'state': state, 'heads': state.heads()}, patch, binary_change]

    # backend.js:96-98
    def save(self, backend):
        return backend_state(backend).save()

    # backend.js:104-107
    def load(self, data):
        state = self.doc_class(data)
        return {'state': state, 'heads': state.heads()}

    # backend.js:116-121
    def loadChanges(self, backend, changes):
        state = backend_state(backend)
        state.apply_changes(list(changes), want_patch=False)
        backend['frozen'] = True
        return {'state': state, 'heads': state.heads()}

    # backend.js:127-129
    def getPatch(self, backend):
        return backend_state(backend).get_patch()

    # backend.js:135-137
    def getHeads(self, backend):
        return backend['heads']

    # backend.js:142-144
    def getAllChanges(self, backend):
        return self.getChanges(backend, [])

    # backend.js:151-156
    def getChanges(self, backend, have_deps):
        if not isinstance(have_deps, (list, tuple)):
            raise TypeError('Pass an array of hashes to Backend.getChanges()')
        return backend_state(backend).get_changes(list(have_deps))

    # backend.js:166-168
    def getChangesAdded(self, backend1, backend2):
        return backend_state(backend2).get_changes_added(backend_state(backend1))

    # backend.js:176-178
    def getChangeByHash(self, backend, hash_):
        return backend_state(backend).get_change_by_hash(hash_)

    # backend.js:190-192
    def getMissingDeps(self, backend, heads=()):
        return backend_state(backend).get_missing_deps(list(heads))
