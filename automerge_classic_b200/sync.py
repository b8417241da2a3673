"""Sync protocol over the native backend — the seven functions backend/index.js re-exports from backend/sync.js.

The reference's sync.js hard-imports the JavaScript backend (sync.js:19), so a replacement backend has to bring these
along (SURVEY.md section 8f, rank 3). This is host-side protocol logic: Bloom filter over change hashes, message and
peer-state encoding, and the two state transitions; every document operation goes through the `Backend` facade
(getHeads / getChanges / getChangeByHash / getMissingDeps / applyChanges), i.e. through the engine. The per-change work
(the Bloom filter of a message, the changes to send) runs on the device when the document offers it (see Sync).

Follows (paths relative to /root/reference): backend/sync.js:24-127 (BloomFilter), :130-227 (wire formats),
:234-306 (makeBloomFilter, getChangesToSend), :308-478 (initSyncState, generateSyncMessage, advanceHeads,
receiveSyncMessage). Hashes are lowercase hex strings, messages and changes are `bytes`, as in the reference.
"""
import hashlib

from .backend import backend_state
from .columnar import inflate_change, uleb
from .engine import Unsupported

HASH_SIZE = 32
MESSAGE_TYPE_SYNC = 0x42      # sync.js:25
PEER_STATE_TYPE = 0x43        # sync.js:26
BITS_PER_ENTRY, NUM_PROBES = 10, 7   # sync.js:31 (1 % false positives; both travel in the wire format)


class _Reader:
    def __init__(self, buf):
        self.buf, self.off = bytes(buf), 0

    def byte(self):
        if self.off >= len(self.buf):
            raise ValueError('buffer ended with incomplete number')
        self.off += 1
        return self.buf[self.off - 1]

    def uint32(self):   # encoding.js:341-363 readUint32
        result, shift = 0, 0
        while self.off < len(self.buf):
            b = self.buf[self.off]
            if shift == 28 and (b & 0xf0) != 0:
                raise ValueError('number out of range')
            result |= (b & 0x7f) << shift
            shift += 7
            self.off += 1
            if not (b & 0x80):
                return result
        raise ValueError('buffer ended with incomplete number')

    def raw(self, n):
        if self.off + n > len(self.buf):
            raise ValueError('subarray exceeds buffer size')
        self.off += n
        return self.buf[self.off - n:self.off]

    def prefixed(self):
        return self.raw(self.uint32())


def _uint32(v):
    if not 0 <= v <= 0xffffffff:
        raise ValueError('number out of range')
    return uleb(v)


class BloomFilter:
    """sync.js:38-127. Entries are SHA-256 hashes already, so the filter does no hashing of its own."""

    def __init__(self, arg):
        if isinstance(arg, (list, tuple)):
            self.num_entries, self.num_bits_per_entry, self.num_probes = len(arg), BITS_PER_ENTRY, NUM_PROBES
            self.bits = bytearray(-(-self.num_entries * self.num_bits_per_entry // 8))
            for h in arg:
                self.add_hash(h)
        elif isinstance(arg, (bytes, bytearray, memoryview)):
            arg = bytes(arg)
            if len(arg) == 0:
                self.num_entries = self.num_bits_per_entry = self.num_probes = 0
                self.bits = bytearray()
            else:
                r = _Reader(arg)
                self.num_entries, self.num_bits_per_entry, self.num_probes = r.uint32(), r.uint32(), r.uint32()
                self.bits = bytearray(r.raw(-(-self.num_entries * self.num_bits_per_entry // 8)))
        else:
            raise TypeError('invalid argument')

    @property
    def bytes(self):
        if self.num_entries == 0:
            return b''
        return _uint32(self.num_entries) + _uint32(self.num_bits_per_entry) + _uint32(self.num_probes) + bytes(self.bits)

    def probes(self, hash_hex):
        """Triple hashing over the first 12 bytes of the hash as three little-endian u32 (sync.js:84-98)."""
        hb = bytes.fromhex(hash_hex)
        if len(hb) != 32:
            raise ValueError('Not a 256-bit hash: %s' % hash_hex)
        modulo = 8 * len(self.bits)
        x = int.from_bytes(hb[0:4], 'little') % modulo
        y = int.from_bytes(hb[4:8], 'little') % modulo
        z = int.from_bytes(hb[8:12], 'little') % modulo
        out = [x]
        for _ in range(1, self.num_probes):
            x = (x + y) % modulo
            y = (y + z) % modulo
            out.append(x)
        return out

    def add_hash(self, hash_hex):
        if len(self.bits) == 0:   # a peer's filter with entries but no bits: the reference computes NaN probes and stores nothing
            return
        for p in self.probes(hash_hex):
            self.bits[p >> 3] |= 1 << (p & 7)

    def contains_hash(self, hash_hex):
        if self.num_entries == 0 or len(self.bits) == 0:   # (sync.js:84-98 with modulo 0: NaN probes, containsHash false: the changes are sent)
            return False
        return all(self.bits[p >> 3] & (1 << (p & 7)) for p in self.probes(hash_hex))


def _encode_hashes(hashes):   # sync.js:130-139
    if not isinstance(hashes, (list, tuple)):
        raise TypeError('hashes must be an array')
    out = bytearray(_uint32(len(hashes)))
    for i, h in enumerate(hashes):
        if i > 0 and hashes[i - 1] >= h:
            raise ValueError('hashes must be sorted')
        hb = bytes.fromhex(h)
        if len(hb) != HASH_SIZE:
            raise TypeError('heads hashes must be 256 bits')
        out += hb
    return bytes(out)


def _decode_hashes(r):   # sync.js:145-151
    return [r.raw(HASH_SIZE).hex() for _ in range(r.uint32())]


def encodeSyncMessage(message):   # sync.js:157-172
    out = bytearray([MESSAGE_TYPE_SYNC])
    out += _encode_hashes(message['heads'])
    out += _encode_hashes(message['need'])
    out += _uint32(len(message['have']))
    for have in message['have']:
        out += _encode_hashes(have['lastSync'])
        out += _uint32(len(have['bloom'])) + bytes(have['bloom'])
    out += _uint32(len(message['changes']))
    for change in message['changes']:
        out += _uint32(len(change)) + bytes(change)
    return bytes(out)


def decodeSyncMessage(data):   # sync.js:177-199 (trailing bytes are ignored: room for protocol extensions)
    r = _Reader(data)
    message_type = r.byte()
    if message_type != MESSAGE_TYPE_SYNC:
        raise ValueError('Unexpected message type: %d' % message_type)
    heads, need = _decode_hashes(r), _decode_hashes(r)
    message = {'heads': heads, 'need': need, 'have': [], 'changes': []}
    for _ in range(r.uint32()):
        last_sync = _decode_hashes(r)
        message['have'].append({'lastSync': last_sync, 'bloom': r.prefixed()})
    for _ in range(r.uint32()):
        message['changes'].append(r.prefixed())
    return message


def initSyncState():   # sync.js:308-317
    return {'sharedHeads': [], 'lastSentHeads': [], 'theirHeads': None, 'theirNeed': None, 'theirHave': None, 'sentHashes': {}}


def encodeSyncState(sync_state):   # sync.js:206-211: only what must survive a reconnect
    return bytes([PEER_STATE_TYPE]) + _encode_hashes(sync_state['sharedHeads'])


def decodeSyncState(data):   # sync.js:217-226
    r = _Reader(data)
    record_type = r.byte()
    if record_type != PEER_STATE_TYPE:
        raise ValueError('Unexpected record type: %d' % record_type)
    state = initSyncState()
    state['sharedHeads'] = _decode_hashes(r)
    return state


def _leb(r):
    result, shift = 0, 0
    while True:
        b = r.byte()
        result |= (b & 0x7f) << shift
        shift += 7
        if not (b & 0x80):
            return result


def _change_meta(change):
    """hash and deps of a binary change (decodeChangeMeta(change, true), columnar.js:778-796)."""
    plain = inflate_change(bytes(change))
    r = _Reader(plain)
    r.raw(8)      # magic bytes + checksum
    r.byte()      # chunk type
    _leb(r)       # chunk length
    deps = [r.raw(32).hex() for _ in range(_leb(r))]
    return {'hash': hashlib.sha256(plain[8:]).hexdigest(), 'deps': deps, 'change': bytes(change)}


class Sync:
    """The sync functions bound to a Backend facade (automerge_classic_b200.Backend or any object with its methods).

    With device=True (the default), the Bloom filter of a message and the choice of the changes to send run in the engine
    when the document has the native methods (GpuBackendDoc.sync_bloom / sync_changes_to_send): from the change hashes it
    already holds, instead of copying, inflating and hashing every change in Python. device=False, a document without
    them (the oracle) or a filter the engine declines keep the host implementation below. Both give the same bytes."""

    def __init__(self, backend_module, device=True):
        self.B = backend_module
        self.device = device

    def _native(self, backend, name):
        if not self.device or not isinstance(backend, dict):
            return None
        fn = getattr(backend.get('state'), name, None)
        if fn is not None:
            backend_state(backend)   # an outdated handle fails as it does in the facade's getChanges
        return fn

    # sync.js:234-238
    def _make_bloom_filter(self, backend, last_sync):
        native = self._native(backend, 'sync_bloom')
        if native is not None and isinstance(last_sync, (list, tuple)):
            return {'lastSync': last_sync, 'bloom': native(list(last_sync))}
        new_changes = self.B.getChanges(backend, last_sync)
        return {'lastSync': last_sync, 'bloom': BloomFilter([_change_meta(c)['hash'] for c in new_changes]).bytes}

    def _changes_to_send(self, backend, have, need):
        """(changes, hashes) of getChangesToSend; hashes is None when the host path chose the changes."""
        native = self._native(backend, 'sync_changes_to_send') if len(have) > 0 else None
        if native is not None:
            last_sync_hashes, bloom_filters = {}, []
            for h in have:
                for x in h['lastSync']:
                    last_sync_hashes[x] = True
                bloom_filters.append(BloomFilter(h['bloom']))   # parsing and its errors stay here
            try:
                return native(list(last_sync_hashes.keys()), bloom_filters, list(need))
            except Unsupported:
                pass   # a filter the device path declines (more than 64 probes): the host path answers
        return self._get_changes_to_send(backend, have, need), None

    # sync.js:246-306
    def _get_changes_to_send(self, backend, have, need):
        if len(have) == 0:
            return [c for c in (self.B.getChangeByHash(backend, h) for h in need) if c is not None]
        last_sync_hashes, bloom_filters = {}, []
        for h in have:
            for x in h['lastSync']:
                last_sync_hashes[x] = True
            bloom_filters.append(BloomFilter(h['bloom']))
        changes = [_change_meta(c) for c in self.B.getChanges(backend, list(last_sync_hashes.keys()))]
        change_hashes, dependents, hashes_to_send = {}, {}, {}
        for change in changes:
            change_hashes[change['hash']] = True
            for dep in change['deps']:
                dependents.setdefault(dep, []).append(change['hash'])
            if all(not bloom.contains_hash(change['hash']) for bloom in bloom_filters):
                hashes_to_send[change['hash']] = True
        stack = list(hashes_to_send.keys())   # everything that depends on a Bloom-negative change goes too
        while stack:
            h = stack.pop()
            for dep in dependents.get(h, ()):
                if dep not in hashes_to_send:
                    hashes_to_send[dep] = True
                    stack.append(dep)
        changes_to_send = []
        for h in need:   # explicitly requested changes
            hashes_to_send[h] = True
            if h not in change_hashes:
                change = self.B.getChangeByHash(backend, h)
                if change is not None:
                    changes_to_send.append(change)
        for change in changes:
            if change['hash'] in hashes_to_send:
                changes_to_send.append(change['change'])
        return changes_to_send

    # sync.js:327-396
    def generateSyncMessage(self, backend, sync_state):
        if not backend:
            raise ValueError('generateSyncMessage called with no Automerge document')
        if not sync_state:
            raise ValueError('generateSyncMessage requires a syncState, which can be created with initSyncState()')
        shared_heads, last_sent_heads = sync_state['sharedHeads'], sync_state['lastSentHeads']
        their_heads, their_need, their_have, sent_hashes = sync_state['theirHeads'], sync_state['theirNeed'], sync_state['theirHave'], sync_state['sentHashes']
        our_heads = list(self.B.getHeads(backend))
        our_need = self.B.getMissingDeps(backend, their_heads or [])
        our_have = []
        if their_heads is None or all(h in their_heads for h in our_need):
            our_have = [self._make_bloom_filter(backend, shared_heads)]
        if their_have:
            last_sync = their_have[0]['lastSync']
            if not all(self.B.getChangeByHash(backend, h) is not None for h in last_sync):
                # the peer's last sync refers to changes we do not have (we lost state): ask for a fresh start
                reset = {'heads': our_heads, 'need': [], 'have': [{'lastSync': [], 'bloom': b''}], 'changes': []}
                return [sync_state, encodeSyncMessage(reset)]
        changes_to_send, hashes = [], []
        if isinstance(their_have, list) and isinstance(their_need, list):
            changes_to_send, hashes = self._changes_to_send(backend, their_have, their_need)
        heads_unchanged = isinstance(last_sent_heads, list) and our_heads == last_sent_heads
        heads_equal = isinstance(their_heads, list) and our_heads == their_heads
        if heads_unchanged and heads_equal and len(changes_to_send) == 0:
            return [sync_state, None]
        if hashes is None:
            hashes = [_change_meta(c)['hash'] for c in changes_to_send]
        keep = [k for k, h in enumerate(hashes) if h not in sent_hashes]
        changes_to_send, hashes = [changes_to_send[k] for k in keep], [hashes[k] for k in keep]
        message = {'heads': our_heads, 'have': our_have, 'need': our_need, 'changes': changes_to_send}
        if changes_to_send:
            sent_hashes = dict(sent_hashes)
            for h in hashes:
                sent_hashes[h] = True
        new_state = dict(sync_state)
        new_state.update({'lastSentHeads': our_heads, 'sentHashes': sent_hashes})
        return [new_state, encodeSyncMessage(message)]

    # sync.js:420-472
    def receiveSyncMessage(self, backend, old_sync_state, binary_message):
        if not backend:
            raise ValueError('generateSyncMessage called with no Automerge document')
        if not old_sync_state:
            raise ValueError('generateSyncMessage requires a syncState, which can be created with initSyncState()')
        shared_heads, last_sent_heads, sent_hashes = old_sync_state['sharedHeads'], old_sync_state['lastSentHeads'], old_sync_state['sentHashes']
        patch = None
        message = decodeSyncMessage(binary_message)
        before_heads = list(self.B.getHeads(backend))
        if message['changes']:
            backend, patch = self.B.applyChanges(backend, message['changes'])
            shared_heads = _advance_heads(before_heads, list(self.B.getHeads(backend)), shared_heads)
        if not message['changes'] and message['heads'] == before_heads:
            last_sent_heads = message['heads']
        known_heads = [h for h in message['heads'] if self.B.getChangeByHash(backend, h) is not None]
        if len(known_heads) == len(message['heads']):
            shared_heads = message['heads']
            if len(message['heads']) == 0:   # the peer has lost all its data: full resync
                last_sent_heads, sent_hashes = [], {}
        else:
            shared_heads = sorted(set(known_heads) | set(shared_heads))
        sync_state = {'sharedHeads': shared_heads, 'lastSentHeads': last_sent_heads, 'theirHave': message['have'],
                      'theirHeads': message['heads'], 'theirNeed': message['need'], 'sentHashes': sent_hashes}
        return [backend, sync_state, patch]


def _advance_heads(my_old_heads, my_new_heads, our_old_shared_heads):   # sync.js:408-413
    new_heads = [h for h in my_new_heads if h not in my_old_heads]
    common_heads = [h for h in our_old_shared_heads if h in my_new_heads]
    return sorted(set(new_heads) | set(common_heads))
