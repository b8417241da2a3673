"""ctypes binding of libamgpu.so (include/amgpu.h) and the document class the Backend facade drives.

`GpuBackendDoc` has the surface of the reference's BackendDoc (backend/new.js:1694-2069): the heavy
lifting — columnar decode, causal gate, op-set ordering, patch computation — runs in the CUDA kernels
behind the C ABI; this module only (1) passes byte buffers across the boundary and (2) inflates the
flat binary patch table into the nested Patch object of @types/automerge/index.d.ts:236-316, which
is what the N-API shim does on the JavaScript side (INTEGRATION.md).

There is no CPU fallback: importing works anywhere, but creating a document raises if libamgpu.so is
missing or no CUDA device is present.
"""
import ctypes as C
import os
import struct

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libamgpu.so')

ACTIONS = ['makeMap', 'set', 'makeList', 'del', 'makeText', 'inc', 'makeTable', 'link']
OBJ_TYPE = {0: 'map', 2: 'list', 4: 'text', 6: 'table'}
PROP_DT = np.dtype([('obj', '<u8'), ('opId', '<u8'), ('keyOff', '<u4'), ('keyLen', '<u4'), ('valLen', '<u4'), ('valOff', '<u4'), ('flags', '<u4'), ('pad', '<u4')])
EDIT_DT = np.dtype([('obj', '<u8'), ('opId', '<u8'), ('index', '<u4'), ('kind', '<u4'), ('valLen', '<u4'), ('valOff', '<u4')])


class AmgError(Exception):
    """Error raised by the engine; `.kind` is the reference's JS error class."""
    KINDS = {1: 'RangeError', 2: 'TypeError', 3: 'Error', 4: 'Unsupported', 5: 'CudaError'}

    def __init__(self, code, msg):
        super().__init__(msg)
        self.code, self.kind, self.message = code, self.KINDS.get(code, 'Error'), msg


class Unsupported(AmgError):
    pass


class _ErrStruct(C.Structure):
    _fields_ = [('code', C.c_int), ('msg', C.c_char * 512)]


class _Bloom(C.Structure):   # amg_bloom: a peer's parsed Bloom filter
    _fields_ = [('num_entries', C.c_uint32), ('num_probes', C.c_uint32), ('bits', C.c_void_p), ('bits_len', C.c_size_t)]


class Library:
    def __init__(self, path):
        if not os.path.exists(path):
            raise RuntimeError('amgpu: %s not found — build it with `python -c "import __graft_entry__ as g; g.build()"` '
                               '(there is no CPU fallback)' % path)
        self.path = path
        L = self.L = C.CDLL(path)
        vp = C.c_void_p
        L.amg_init.restype = vp
        L.amg_init.argtypes = [C.c_int, vp]
        L.amg_load.restype = vp
        L.amg_load.argtypes = [C.c_int, vp, C.c_size_t, vp]
        L.amg_clone.restype = vp
        L.amg_clone.argtypes = [vp, vp]
        L.amg_free.argtypes = [vp]
        L.amg_patch_bytes.restype = vp
        L.amg_patch_bytes.argtypes = [vp, vp]
        L.amg_patch_free.argtypes = [vp]
        L.amg_arena.restype = vp
        L.amg_arena.argtypes = [vp, vp]
        L.amg_buffers_count.restype = C.c_size_t
        L.amg_buffers_count.argtypes = [vp]
        L.amg_buffers_get.restype = vp
        L.amg_buffers_get.argtypes = [vp, C.c_size_t, vp]
        L.amg_buffers_free.argtypes = [vp]
        L.amg_kernel_launches.restype = C.c_uint64
        L.amg_kernel_launches.argtypes = [vp]
        L.amg_free_mem.argtypes = [vp]
        for name in ('amg_apply_changes', 'amg_apply_changes_packed', 'amg_get_patch', 'amg_get_state', 'amg_get_heads', 'amg_get_changes',
                     'amg_get_changes_added', 'amg_get_change_by_hash', 'amg_get_missing_deps', 'amg_clock_of', 'amg_hash_by_actor',
                     'amg_debug_dump_ops', 'amg_debug_decode', 'amg_debug_decode_column', 'amg_bench_decode', 'amg_last_timings',
                     'amg_sync_bloom', 'amg_sync_changes_to_send'):
            getattr(L, name).restype = C.c_int
        L.amg_sync_bloom.argtypes = [vp, vp, C.c_size_t, vp, vp]
        L.amg_sync_changes_to_send.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, vp, C.c_size_t, vp, vp, vp]
        L.amg_decode_changes.restype = C.c_int
        L.amg_decode_changes.argtypes = [vp, vp, vp, C.c_size_t, vp, vp, vp]
        L.amg_decode_history.restype = C.c_int
        L.amg_decode_history.argtypes = [vp, vp, vp]
        L.amg_encode_changes.restype = C.c_int
        L.amg_encode_changes.argtypes = [vp, vp, C.c_size_t, vp, vp, vp, vp]
        L.amg_get_history_patches.restype = C.c_int
        L.amg_get_history_patches.argtypes = [vp, vp, C.c_size_t, vp, vp]
        L.amg_merge.restype = C.c_int
        L.amg_merge.argtypes = [vp, vp, C.c_int, vp, vp]
        L.amg_merge_many.restype = C.c_int
        L.amg_merge_many.argtypes = [vp, vp, C.c_size_t, C.c_int, vp, vp]
        L.amg_apply_local_change.restype = C.c_int
        L.amg_apply_local_change.argtypes = [vp, vp, C.c_size_t, C.c_int, vp, vp, vp]
        L.amg_clock_of.argtypes = [vp, vp, C.c_size_t, vp, vp]
        for name in ('amg_last_sync_ms', 'amg_last_decode_ms', 'amg_last_encode_ms', 'amg_last_history_ms', 'amg_last_merge_ms', 'amg_last_local_ms',
                     'amg_last_graph_ms'):
            getattr(L, name).restype = C.c_float
            getattr(L, name).argtypes = [vp]

    def check(self, rc, err):
        if rc != 0:
            msg = err.msg.decode('utf-8', 'replace')
            raise (Unsupported if rc == 4 else AmgError)(rc, msg)

    def check_indexed(self, rc, err, failed):
        """check() for a call over a batch of changes: the error carries `.failed_index`, the change it names"""
        try:
            self.check(rc, err)
        except AmgError as e:
            e.failed_index = failed.value
            raise


def _as_buffer(blob):
    """bytes / bytearray (copied), a numpy array, or a ctypes pointer / address (e.g. pinned host or device memory) as a
    pointer argument"""
    if isinstance(blob, (bytes, bytearray)):
        return (C.c_uint8 * max(len(blob), 1)).from_buffer_copy(bytes(blob) if len(blob) else b'\0')   # (an empty list of changes is legal)
    if isinstance(blob, np.ndarray):
        return blob.ctypes.data_as(C.c_void_p)
    return blob


_default = None


def default_library():
    global _default
    if _default is None:
        _default = Library(LIB_PATH)
    return _default


def decode_value(val_len, raw):
    """reference columnar.js:300-329 decodeValue -> patch value dict {'type':'value','value':..,['datatype':..]}"""
    tag = val_len & 15
    if val_len == 0:
        return {'type': 'value', 'value': None}
    if val_len == 1:
        return {'type': 'value', 'value': False}
    if val_len == 2:
        return {'type': 'value', 'value': True}
    if tag == 6:
        return {'type': 'value', 'value': bytes(raw).decode('utf-8', 'replace')}
    if tag in (3, 4, 8, 9):
        v, shift = 0, 0
        for b in raw:
            v |= (b & 0x7f) << shift
            shift += 7
            if not b & 0x80:
                if tag != 3 and b & 0x40:
                    v -= 1 << shift
                break
        return {'type': 'value', 'value': v, 'datatype': {3: 'uint', 4: 'int', 8: 'counter', 9: 'timestamp'}[tag]}
    if tag == 5:
        if len(raw) != 8:
            raise AmgError(1, 'Invalid length for floating point number: %d' % len(raw))
        return {'type': 'value', 'value': struct.unpack('<d', bytes(raw))[0], 'datatype': 'float64'}
    return {'type': 'value', 'value': bytes(raw), 'datatype': tag}


def empty_object_patch(object_id, action):
    t = OBJ_TYPE.get(action)
    if t in ('list', 'text'):
        return {'objectId': object_id, 'type': t, 'edits': []}
    return {'objectId': object_id, 'type': t, 'props': {}}


class FlatPatch:
    """Zero-copy view of the flat patch table (layout in include/amgpu.h)."""

    def __init__(self, raw):
        self.raw = self.arena = raw   # keyOff / valOff of the records index the patch buffer itself (its bytes section)
        h = self.hdr = np.frombuffer(raw, dtype='<u8', count=20)
        assert int(h[0]) == 0x31504747414d41, 'bad patch magic'
        self.max_op, self.pending = int(h[1]), int(h[2])
        self.actor_seq = None
        if int(h[3]):
            self.actor_seq = (bytes(raw[int(h[5]):int(h[5]) + int(h[6])]).hex(), int(h[4]))
        self.actors, off = [], int(h[7])
        for _ in range(int(h[8])):
            ln = struct.unpack_from('<I', raw, off)[0]
            self.actors.append(bytes(raw[off + 4:off + 4 + ln]).hex())
            off += 4 + ln
            off += (-off) % 4
        ck = np.frombuffer(raw, dtype='<u8', count=2 * int(h[10]), offset=int(h[9])).reshape(-1, 2)
        self.clock = {self.actors[int(a)]: int(s) for a, s in ck}
        self.deps = [bytes(raw[int(h[11]) + 32 * i:int(h[11]) + 32 * i + 32]).hex() for i in range(int(h[12]))]
        self.props = np.frombuffer(raw, dtype=PROP_DT, count=int(h[14]), offset=int(h[13]))
        self.edits = np.frombuffer(raw, dtype=EDIT_DT, count=int(h[16]), offset=int(h[15]))
        # elemOff == 0: the section is not shipped because every insert's elemId equals its opId
        self.edit_elem = np.frombuffer(raw, dtype='<u8', count=int(h[16]), offset=int(h[17])) if int(h[17]) else self.edits['opId']

    def op_id(self, x):
        x = int(x)
        return '%d@%s' % (x >> 16, self.actors[x & 0xffff])

    def header(self):
        out = {'maxOp': self.max_op, 'clock': self.clock, 'deps': self.deps, 'pendingChanges': self.pending}
        if self.actor_seq:
            out['actor'], out['seq'] = self.actor_seq
        return out

    def to_patch(self, whole_doc):
        """Assembles the nested Patch (what the N-API shim does in JS)."""
        arena = self.arena
        patches = {'_root': {'objectId': '_root', 'type': 'map', 'props': {}}}
        # pass 1: every object that appears as a value gets its (empty) patch
        for rec in self.props:
            action = int(rec['flags']) >> 8
            if action % 2 == 0 and not int(rec['flags']) & 1:
                oid = self.op_id(rec['opId'])
                patches.setdefault(oid, empty_object_patch(oid, action))
        for rec in self.edits:
            action = int(rec['kind']) >> 16
            if action % 2 == 0 and (int(rec['kind']) & 0xff) != 1:
                oid = self.op_id(rec['opId'])
                patches.setdefault(oid, empty_object_patch(oid, action))
        # pass 2: map entries
        for rec in self.props:
            obj = '_root' if int(rec['obj']) == 0 else self.op_id(rec['obj'])
            p = patches.get(obj)
            if p is None or 'props' not in p:
                continue   # object not reachable from the root (its make op is no longer visible)
            key = bytes(arena[int(rec['keyOff']):int(rec['keyOff']) + int(rec['keyLen'])]).decode('utf-8', 'replace')
            flags = int(rec['flags'])
            action = flags >> 8
            if flags & 1:
                p['props'].setdefault(key, {})
            elif action == 1 and flags & 2:     # counter: the engine summed the increments (new.js:941-966)
                total = int(rec['valOff']) | (int(rec['pad']) << 32)
                total -= (1 << 64) if total >= (1 << 63) else 0
                p['props'].setdefault(key, {})[self.op_id(rec['opId'])] = {'type': 'value', 'value': total, 'datatype': 'counter'}
            elif action == 1:
                vl, vo = int(rec['valLen']), int(rec['valOff'])
                p['props'].setdefault(key, {})[self.op_id(rec['opId'])] = decode_value(vl, arena[vo:vo + (vl >> 4)])
            elif action % 2 == 0:
                oid = self.op_id(rec['opId'])
                p['props'].setdefault(key, {})[oid] = patches[oid]
            elif not whole_doc:
                p['props'].setdefault(key, {})
        # pass 3: list edits (already ordered per object; runs flagged by the RunFlag kernel)
        for j, rec in enumerate(self.edits):
            obj = self.op_id(rec['obj'])
            p = patches.get(obj)
            if p is None or 'edits' not in p:
                continue
            edits = p['edits']
            kind, run_start, multi, action = int(rec['kind']) & 0xff, bool(int(rec['kind']) & 0x100), bool(int(rec['kind']) & 0x200), int(rec['kind']) >> 16
            index = int(rec['index'])
            if kind == 1:
                if run_start:
                    edits.append({'action': 'remove', 'index': index, 'count': 1})
                else:
                    edits[-1]['count'] += 1
                continue
            if action == 1 and int(rec['kind']) & 0x1000:   # counter with increments: the engine summed them (new.js:941-966)
                total = int(rec['valLen']) | (int(rec['valOff']) << 32)
                total -= (1 << 64) if total >= (1 << 63) else 0
                value = {'type': 'value', 'value': total, 'datatype': 'counter'}
            elif action == 1:
                vl, vo = int(rec['valLen']), int(rec['valOff'])
                value = decode_value(vl, arena[vo:vo + (vl >> 4)])
            elif action % 2 == 0:
                value = patches[self.op_id(rec['opId'])]
            else:
                continue
            if kind == 2:
                edits.append({'action': 'update', 'index': index, 'opId': self.op_id(rec['opId']), 'value': value})
            elif not run_start:
                edits[-1]['values'].append(value['value'])     # continues the multi-insert opened by an earlier record
            elif multi:
                edit = {'action': 'multi-insert', 'index': index, 'elemId': self.op_id(self.edit_elem[j]), 'values': [value['value']]}
                if value.get('datatype'):
                    edit['datatype'] = value['datatype']
                edits.append(edit)
            else:
                edits.append({'action': 'insert', 'index': index, 'elemId': self.op_id(self.edit_elem[j]), 'opId': self.op_id(rec['opId']), 'value': value})
        out = self.header()
        out['diffs'] = patches['_root']
        return out


NULL32 = 0xffffffff
CHANGE_DT = np.dtype([('hash', 'u1', 32), ('seq', '<u8'), ('startOp', '<u8'), ('time', '<i8'), ('msgOff', '<u4'), ('msgLen', '<u4'),
                      ('depsOff', '<u4'), ('nDeps', '<u4'), ('actorFirst', '<u4'), ('nActors', '<u4'), ('extraOff', '<u4'), ('extraLen', '<u4'),
                      ('hasExtra', '<u4'), ('pad', '<u4'), ('firstOp', '<u8'), ('nOps', '<u8'), ('firstPred', '<u8'), ('nPreds', '<u8')])
OP_DT = np.dtype([(f, '<u4') for f in ('objActor', 'objCtr', 'keyActor', 'keyCtr', 'keyStrOff', 'keyStrLen', 'insert', 'action', 'valLen', 'valOff',
                                       'chldActor', 'chldCtr', 'predFirst', 'predNum', 'change', 'pad')])
PRED_DT = np.dtype([('actor', '<u4'), ('ctr', '<u4')])
ACTOR_DT = np.dtype([('off', '<u4'), ('len', '<u4')])


class FlatChanges:
    """Zero-copy view of a change table (amg_decode_changes / amg_decode_history; layout in include/amgpu.h)."""

    def __init__(self, raw):
        self.raw = raw
        h = self.hdr = np.frombuffer(raw, dtype='<u8', count=12)
        assert int(h[0]) == 0x31474843474d41, 'bad change table magic'
        self.changes = np.frombuffer(raw, dtype=CHANGE_DT, count=int(h[1]), offset=int(h[2]))
        self.ops = np.frombuffer(raw, dtype=OP_DT, count=int(h[3]), offset=int(h[4]))
        self.preds = np.frombuffer(raw, dtype=PRED_DT, count=int(h[5]), offset=int(h[6]))
        self.actors = np.frombuffer(raw, dtype=ACTOR_DT, count=int(h[7]), offset=int(h[8]))

    def __len__(self):
        return len(self.changes)

    @classmethod
    def from_changes(cls, changes):
        """The inverse of to_changes(): the change table of a list of change dicts (the form columnar.encode_change takes).
        Multi-ops are expanded, op ids parsed and values encoded by columnar's expand_multi_ops / parse_op_id / encode_value,
        which raise their errors for what is wrong at the dict level; everything else is checked by the encoder. Each change's
        actor table lists its actors in first-use order (the encoder writes the canonical one); preds and deps keep their order."""
        from .columnar import expand_multi_ops, parse_op_id as _parse, encode_value, hex_bytes, ACTIONS as ACTION_NAMES

        def parse_op_id(s):   # the table's counters are 32-bit, and 0xffffffff is its null
            ctr, actor = _parse(s)
            if ctr >= NULL32:
                raise Unsupported(4, "amgpu: an operation counter beyond the change table's 32-bit fields: %s" % s)
            return ctr, actor
        blob = bytearray()   # the bytes section; offsets are relative to it until the layout is known

        def put(b):
            off = len(blob)
            blob.extend(b)
            return off
        ch_cols = {f: [] for f in ('seq', 'startOp', 'time', 'msgOff', 'msgLen', 'depsOff', 'nDeps', 'actorFirst', 'nActors',
                                   'extraOff', 'extraLen', 'hasExtra', 'firstOp', 'nOps', 'firstPred', 'nPreds')}
        ops, preds, actors = [], [], []
        for change in changes:
            author = change['actor']
            ids, order = {author: 0}, [author]

            def num(a):
                if a not in ids:
                    ids[a] = len(order)
                    order.append(a)
                return ids[a]
            first_op, first_pred = len(ops), len(preds)
            for op in expand_multi_ops(change['ops'], change['startOp'], author):
                if op['obj'] == '_root':
                    oa = oc = NULL32
                else:
                    oc, a = parse_op_id(op['obj'])
                    oa = num(a)
                ka = kc = ks_off = ks_len = NULL32
                if op.get('key'):
                    k = op['key'].encode('utf-8')
                    ks_off, ks_len = put(k), len(k)
                elif op.get('elemId') == '_head':
                    kc = 0
                elif op.get('elemId') is not None:
                    kc, a = parse_op_id(op['elemId'])
                    if kc == 0:   # a counter-0 element id is not _head (columnar.js:193): the table cannot hold it
                        raise ValueError('Unexpected operation key: %r' % (op,))
                    ka = num(a)
                act = op.get('action')
                if act in ACTION_NAMES:
                    act = ACTION_NAMES.index(act)
                elif not isinstance(act, int):
                    raise ValueError('Unexpected operation action: %r' % (act,))
                val_len, raw = [], bytearray()
                encode_value(op, val_len, raw)
                ca = cc = NULL32
                if op.get('child'):
                    cc, a = parse_op_id(op['child'])
                    ca = num(a)
                p0 = len(preds)
                for p in op.get('pred', []):
                    c, a = parse_op_id(p)
                    preds.append((num(a), c))
                ops.append((oa, oc, ka, kc, ks_off, ks_len, 1 if op.get('insert') else 0, act, val_len[0], put(raw), ca, cc,
                            p0, len(preds) - p0, len(ch_cols['seq']), 0))
            deps = [hex_bytes(d) for d in change.get('deps', [])]
            if any(len(d) != 32 for d in deps):
                raise ValueError('a dependency is not a 32-byte hash')
            msg = (change.get('message') or '').encode('utf-8')
            extra = bytes(change.get('extraBytes') or b'')
            for k, v in (('seq', change['seq']), ('startOp', change['startOp']), ('time', change.get('time', 0)),
                         ('msgOff', put(msg)), ('msgLen', len(msg)), ('depsOff', put(b''.join(deps))), ('nDeps', len(deps)),
                         ('actorFirst', len(actors)), ('nActors', len(order)), ('extraOff', put(extra)), ('extraLen', len(extra)),
                         ('hasExtra', 1 if extra else 0), ('firstOp', first_op), ('nOps', len(ops) - first_op),
                         ('firstPred', first_pred), ('nPreds', len(preds) - first_pred)):
                ch_cols[k].append(v)
            for a in order:
                b = hex_bytes(a)
                actors.append((put(b), len(b)))
        n, M, P, A = len(ch_cols['seq']), len(ops), len(preds), len(actors)
        changes_off = 96
        ops_off = changes_off + n * CHANGE_DT.itemsize
        preds_off = ops_off + M * OP_DT.itemsize
        actors_off = preds_off + P * PRED_DT.itemsize
        bytes_off = actors_off + A * ACTOR_DT.itemsize
        size = (bytes_off + len(blob) + 7) & ~7
        raw = bytearray(size)
        np.frombuffer(raw, dtype='<u8', count=12)[:] = [0x31474843474d41, n, changes_off, M, ops_off, P, preds_off, A, actors_off,
                                                        bytes_off, len(blob), 0]
        ch = np.frombuffer(raw, dtype=CHANGE_DT, count=n, offset=changes_off)
        for k, v in ch_cols.items():
            ch[k] = v
        for k in ('msgOff', 'depsOff', 'extraOff'):
            ch[k] += bytes_off
        if M:
            o = np.frombuffer(raw, dtype=OP_DT, count=M, offset=ops_off)
            o[:] = np.array(ops, dtype=np.uint32).view(OP_DT).reshape(M)
            for k, nk in (('keyStrOff', 'keyStrLen'), ('valOff', None)):
                sel = o[nk] != NULL32 if nk else slice(None)
                o[k][sel] += bytes_off
        if P:
            np.frombuffer(raw, dtype=PRED_DT, count=P, offset=preds_off)[:] = np.array(preds, dtype=np.uint32).view(PRED_DT).reshape(P)
        if A:
            a = np.frombuffer(raw, dtype=ACTOR_DT, count=A, offset=actors_off)
            a[:] = np.array(actors, dtype=np.uint32).view(ACTOR_DT).reshape(A)
            a['off'] += bytes_off
        raw[bytes_off:bytes_off + len(blob)] = blob
        return cls(bytes(raw))

    def hashes(self):
        return [bytes(h).hex() for h in self.changes['hash']]

    def to_changes(self):
        """The dicts columnar.decode_change returns (columnar.js:770-776 decodeChange), one per change."""
        from .columnar import decode_value, ACTIONS as ACTION_NAMES
        raw, out = self.raw, []
        ops, preds, actor_refs = self.ops.tolist(), self.preds.tolist(), self.actors.tolist()
        for rec in self.changes:
            a0, na = int(rec['actorFirst']), int(rec['nActors'])
            actors = [bytes(raw[o:o + ln]).hex() for o, ln in actor_refs[a0:a0 + na]]
            d0 = int(rec['depsOff'])
            mo = int(rec['msgOff'])
            change = {'actor': actors[0], 'seq': int(rec['seq']), 'startOp': int(rec['startOp']), 'time': int(rec['time']),
                      'message': bytes(raw[mo:mo + int(rec['msgLen'])]).decode('utf-8', 'replace'),
                      'deps': [bytes(raw[d0 + 32 * k:d0 + 32 * k + 32]).hex() for k in range(int(rec['nDeps']))]}
            if int(rec['hasExtra']):
                eo = int(rec['extraOff'])
                change['extraBytes'] = bytes(raw[eo:eo + int(rec['extraLen'])])

            def actor(i):
                return None if i == NULL32 else actors[i]

            def num(v):
                return None if v == NULL32 else v
            change_ops = []
            f0 = int(rec['firstOp'])
            for (obj_a, obj_c, key_a, key_c, ks_off, ks_len, insert, action, val_len, val_off, ch_a, ch_c, p0, pn, _, _) in ops[f0:f0 + int(rec['nOps'])]:
                obj = '_root' if obj_c == NULL32 else '%d@%s' % (obj_c, actor(obj_a))
                act = None if action == NULL32 else (ACTION_NAMES[action] if action < len(ACTION_NAMES) else action)
                key = None if ks_len == NULL32 else bytes(raw[ks_off:ks_off + ks_len]).decode('utf-8', 'replace')
                if key:
                    op = {'obj': obj, 'key': key, 'action': act}
                else:
                    op = {'obj': obj, 'elemId': '_head' if key_c == 0 else '%s@%s' % (num(key_c), actor(key_a)), 'action': act}
                op['insert'] = bool(insert)
                tag = 0 if val_len == NULL32 else val_len
                if act in ('set', 'inc'):
                    value, datatype = decode_value(tag, raw[val_off:val_off + (tag >> 4)])
                    op['value'] = value
                    if datatype:
                        op['datatype'] = datatype
                if ch_c != NULL32:
                    op['child'] = '%d@%s' % (ch_c, actor(ch_a))
                op['pred'] = ['%s@%s' % (num(c), actor(a)) for a, c in preds[p0:p0 + pn]]
                change_ops.append(op)
            change['ops'] = change_ops
            change['hash'] = bytes(rec['hash']).hex()
            out.append(change)
        return out


class GpuBackendDoc:
    """BackendDoc (backend/new.js:1694) over the CUDA engine."""
    _library = None   # tests may bind a subclass to another build of the same sources

    @classmethod
    def lib(cls):
        return cls._library or default_library()

    def __init__(self, data=None, _handle=None, device=0):
        self._lib = self.lib()
        L = self._lib.L
        if _handle is not None:
            self.h = _handle
            return
        err = _ErrStruct()
        dev = int(os.environ.get('AMG_DEVICE', device))
        if data is not None:
            data = bytes(data)
            h = L.amg_load(dev, data, C.c_size_t(len(data)), C.byref(err))
        else:
            h = L.amg_init(dev, C.byref(err))
        if not h:
            raise (Unsupported if err.code == 4 else AmgError)(err.code, err.msg.decode('utf-8', 'replace'))
        self.h = C.c_void_p(h)

    def __del__(self):
        try:
            if getattr(self, 'h', None):
                self._lib.L.amg_free(self.h)
                self.h = None
        except Exception:
            pass

    # ---- helpers
    def _arena(self):
        n = C.c_size_t()
        p = self._lib.L.amg_arena(self.h, C.byref(n))
        if not p or n.value == 0:
            return memoryview(b'')
        return memoryview((C.c_uint8 * n.value).from_address(p)).cast('B')

    def _take_patch(self, pp):
        n = C.c_size_t()
        p = self._lib.L.amg_patch_bytes(pp, C.byref(n))
        raw = bytes((C.c_uint8 * n.value).from_address(p))
        self._lib.L.amg_patch_free(pp)
        return FlatPatch(raw)

    def _buffers(self, bl):
        L = self._lib.L
        out = []
        for i in range(L.amg_buffers_count(bl)):
            n = C.c_size_t()
            p = L.amg_buffers_get(bl, i, C.byref(n))
            out.append(C.string_at(p, n.value) if n.value else b'')
        L.amg_buffers_free(bl)
        return out

    # ---- BackendDoc surface
    def clone(self):
        err = _ErrStruct()
        h = self._lib.L.amg_clone(self.h, C.byref(err))
        if not h:
            raise AmgError(err.code, err.msg.decode('utf-8', 'replace'))
        return type(self)(_handle=C.c_void_p(h))

    def apply_changes_flat(self, changes, is_local=False, want_patch=True):
        n = len(changes)
        blob = b''.join(bytes(c) for c in changes)
        offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum([len(c) for c in changes], out=offs[1:])
        return self.apply_packed_flat(blob, offs, n, is_local, want_patch)

    def apply_packed_flat(self, blob, offs, n, is_local=False, want_patch=True):
        pp, err = C.c_void_p(), _ErrStruct()
        rc = self._lib.L.amg_apply_changes_packed(self.h, _as_buffer(blob), offs.ctypes.data_as(C.c_void_p), C.c_size_t(n), int(is_local), int(want_patch),
                                                  C.byref(pp), C.byref(err))
        self._lib.check(rc, err)
        return self._take_patch(pp) if want_patch else None

    def apply_changes_ptrs_flat(self, changes, is_local=False, want_patch=True):
        """amg_apply_changes: one pointer + length per change (what an N-API binding passes for a Uint8Array[])."""
        n = len(changes)
        keep = [bytes(c) for c in changes]
        bufs = (C.c_char_p * max(n, 1))(*keep)
        lens = (C.c_size_t * max(n, 1))(*[len(c) for c in keep])
        pp, err = C.c_void_p(), _ErrStruct()
        fn = self._lib.L.amg_apply_changes
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        rc = fn(self.h, bufs, lens, C.c_size_t(n), int(is_local), int(want_patch), C.byref(pp), C.byref(err))
        self._lib.check(rc, err)
        return self._take_patch(pp) if want_patch else None

    def apply_changes(self, changes, is_local=False, want_patch=True):
        if isinstance(changes, (bytes, bytearray)):
            raise TypeError('applyChanges takes an array of Uint8Arrays, not just a single Uint8Array')
        fp = self.apply_changes_flat(list(changes), is_local, want_patch)
        return fp.to_patch(False) if want_patch else None

    def get_patch_flat(self):
        pp, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_patch(self.h, C.byref(pp), C.byref(err)), err)
        return self._take_patch(pp)

    def get_patch(self):
        return self.get_patch_flat().to_patch(True)

    def _state(self):
        pp, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_state(self.h, C.byref(pp), C.byref(err)), err)
        return self._take_patch(pp)

    def heads(self):
        return self._state().deps

    def clock(self):
        return self._state().clock

    def max_op(self):
        return self._state().max_op

    def save(self):
        """Backend.save (new.js:2033-2055): the document chunk, columns encoded on the device."""
        fn = getattr(self._lib.L, 'amg_save', None)
        if fn is None:
            raise Unsupported(4, 'amgpu: this build of libamgpu has no amg_save')
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(fn(self.h, C.byref(bl), C.byref(err)), err)
        return self._buffers(bl)[0]

    def clock_of(self, actor):
        """clock[actor] (0 for an actor the document has not seen), without building the whole clock"""
        a = bytes.fromhex(actor)
        seq, err = C.c_uint64(), _ErrStruct()
        self._lib.check(self._lib.L.amg_clock_of(self.h, a, C.c_size_t(len(a)), C.byref(seq), C.byref(err)), err)
        return seq.value

    def hash_by_actor(self, actor, index):
        a = bytes.fromhex(actor)
        out, found, err = (C.c_uint8 * 32)(), C.c_int(), _ErrStruct()
        self._lib.check(self._lib.L.amg_hash_by_actor(self.h, a, C.c_size_t(len(a)), C.c_uint64(index), out, C.byref(found), C.byref(err)), err)
        return bytes(out).hex() if found.value else None

    def get_changes(self, have_deps):
        deps = b''.join(bytes.fromhex(h) for h in have_deps)
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_changes(self.h, deps, C.c_size_t(len(have_deps)), C.byref(bl), C.byref(err)), err)
        return self._buffers(bl)

    def get_changes_added(self, old):
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_changes_added(self.h, old.h, C.byref(bl), C.byref(err)), err)
        return self._buffers(bl)

    def merge_flat(self, other, want_patch=True):
        """amg_merge: applies the changes of `other` this document lacks, in getChangesAdded order, copied device to device
        (src/automerge.js:61-67). Returns the FlatPatch applyChanges would (None with want_patch=False). Raises
        Unsupported when the documents are on different devices, before anything changed."""
        pp, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_merge(self.h, other.h, int(want_patch), C.byref(pp), C.byref(err)), err)
        return self._take_patch(pp) if want_patch else None

    def merge(self, other, want_patch=True):
        """merge_flat as the patch dict applyChanges returns."""
        fp = self.merge_flat(other, want_patch)
        return fp.to_patch(False) if want_patch else None

    def merge_many_flat(self, others, want_patch=True):
        """amg_merge_many: merge_flat folded over `others` in one apply. Applies the changes of each document this one and
        the earlier ones lack, each remote's in getChangesAdded order; a change several remotes hold goes over once, from
        the first. Returns the FlatPatch applyChanges would return for that list (None with want_patch=False). Raises
        Unsupported when a document is on another device, before anything changed."""
        hs = (C.c_void_p * max(len(others), 1))(*[o.h for o in others])
        pp, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_merge_many(self.h, hs, C.c_size_t(len(others)), int(want_patch), C.byref(pp), C.byref(err)), err)
        return self._take_patch(pp) if want_patch else None

    def merge_many(self, others, want_patch=True):
        """merge_many_flat as the patch dict applyChanges returns."""
        fp = self.merge_many_flat(others, want_patch)
        return fp.to_patch(False) if want_patch else None

    def last_merge_ms(self):
        """Device span of the last merge_flat or merge_many_flat call (CUDA events), ms."""
        return float(self._lib.L.amg_last_merge_ms(self.h))

    # ---- applyLocalChange (backend.js:54-91), on the device
    def apply_local_change_flat(self, change, want_patch=True):
        """amg_apply_local_change: the change request (a change dict, as encode_change takes it) encoded with the author's
        previous change hash added to its deps, and applied. Returns (FlatPatch without the new change's hash in its deps,
        or None with want_patch=False; the binary change as encodeChange returns it). Raises Unsupported before anything
        changed for a request the change table cannot hold (a counter of 2^32 or more)."""
        table = FlatChanges.from_changes([change]).raw
        pp, bl, err = C.c_void_p(), C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_apply_local_change(self.h, C.cast(C.c_char_p(table), C.c_void_p), C.c_size_t(len(table)), int(want_patch),
                                                           C.byref(pp), C.byref(bl), C.byref(err)), err)
        return (self._take_patch(pp) if want_patch else None), self._buffers(bl)[0]

    def apply_local_change(self, change):
        """apply_local_change_flat with the patch as the dict applyChanges returns."""
        fp, binary = self.apply_local_change_flat(change)
        return fp.to_patch(False), binary

    def last_local_ms(self):
        """Device span of the last apply_local_change_flat call (CUDA events), ms."""
        return float(self._lib.L.amg_last_local_ms(self.h))

    def get_change_by_hash(self, hash_):
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_change_by_hash(self.h, bytes.fromhex(hash_), C.byref(bl), C.byref(err)), err)
        got = self._buffers(bl)
        return got[0] if got else None

    def get_missing_deps(self, heads=()):
        hs = b''.join(bytes.fromhex(h) for h in heads)
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_missing_deps(self.h, hs, C.c_size_t(len(heads)), C.byref(bl), C.byref(err)), err)
        return [b.hex() for b in self._buffers(bl)]

    def last_graph_ms(self):
        """Device span of the last get_changes / get_change_by_hash / get_missing_deps / hash_by_actor call (CUDA events), ms."""
        return float(self._lib.L.amg_last_graph_ms(self.h))

    # ---- sync protocol (automerge_classic_b200/sync.py uses these when the document has them)
    def sync_bloom(self, last_sync):
        """makeBloomFilter(backend, lastSync) (sync.js:234-238): BloomFilter([hashes of getChanges(lastSync)]).bytes, built on
        the device from the hashes the engine holds."""
        hs = b''.join(bytes.fromhex(h) for h in last_sync)
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_sync_bloom(self.h, hs, C.c_size_t(len(last_sync)), C.byref(bl), C.byref(err)), err)
        return self._buffers(bl)[0]

    def sync_changes_to_send(self, last_sync, filters, need):
        """getChangesToSend(backend, have, need) for a non-empty `have` (sync.js:246-306). last_sync: the union of the
        have entries' lastSync hashes in first-seen order; filters: parsed Bloom filters (objects with num_entries,
        num_probes and bits, like sync.BloomFilter). Returns (changes, hashes): the changes to send in the reference's
        order and their hashes (hex). Raises Unsupported for a filter with more than 64 probes."""
        hs = b''.join(bytes.fromhex(h) for h in last_sync)
        nd = b''.join(bytes.fromhex(h) for h in need)
        keep = [bytes(f.bits) for f in filters]   # alive until the call returns
        arr = (_Bloom * max(len(filters), 1))()
        for i, (f, bits) in enumerate(zip(filters, keep)):
            arr[i].num_entries, arr[i].num_probes, arr[i].bits_len = f.num_entries, f.num_probes, len(bits)
            arr[i].bits = C.cast(C.c_char_p(bits), C.c_void_p) if bits else None
        bc, bh, err = C.c_void_p(), C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_sync_changes_to_send(self.h, hs, C.c_size_t(len(last_sync)), arr, C.c_size_t(len(filters)),
                                                             nd, C.c_size_t(len(need)), C.byref(bc), C.byref(bh), C.byref(err)), err)
        hx = self._buffers(bh)[0].hex()
        return self._buffers(bc), [hx[i:i + 64] for i in range(0, len(hx), 64)]

    def last_sync_ms(self):
        """Device span of the last sync_bloom / sync_changes_to_send call (CUDA events), ms."""
        return float(self._lib.L.amg_last_sync_ms(self.h))

    # ---- decodeChange / decodeChanges (columnar.js:770-776), on the device
    def decode_packed_flat(self, blob, offs, n):
        """amg_decode_changes over change i = blob[offs[i]:offs[i+1]] (bytes, a numpy array, or a pointer to pinned or device
        memory). Raises AmgError with `.failed_index` = the change the reference fails on first."""
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        bl, failed, err = C.c_void_p(), C.c_size_t(), _ErrStruct()
        rc = self._lib.L.amg_decode_changes(self.h, _as_buffer(blob), offs.ctypes.data_as(C.c_void_p), C.c_size_t(n), C.byref(bl), C.byref(failed), C.byref(err))
        self._lib.check_indexed(rc, err, failed)
        return FlatChanges(self._buffers(bl)[0])

    def decode_changes_flat(self, changes):
        """decodeChange of every binary change in `changes` (chunk type 1 or 2), in one device call: a FlatChanges view.
        The document is not touched."""
        n = len(changes)
        offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum([len(c) for c in changes], out=offs[1:])
        return self.decode_packed_flat(b''.join(bytes(c) for c in changes), offs, n)

    def decode_history_flat(self):
        """decodeChanges(getAllChanges()) of this document, read from device memory: a FlatChanges view."""
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_decode_history(self.h, C.byref(bl), C.byref(err)), err)
        return FlatChanges(self._buffers(bl)[0])

    def last_decode_ms(self):
        """Device span of the last decode_*_flat call (CUDA events), ms."""
        return float(self._lib.L.amg_last_decode_ms(self.h))

    # ---- encodeChange (columnar.js:710-739), on the device
    def encode_flat(self, table, length=None):
        """amg_encode_changes: encodeChange of every change of a change table - a FlatChanges, the table's bytes, a numpy array
        or a pointer (int) to pinned or device memory with `length`. Returns (binary changes, hashes as hex strings); the
        document is not touched. Raises AmgError with `.failed_index` = the first failing change."""
        if isinstance(table, FlatChanges):
            table = table.raw
        if isinstance(table, bytes):
            n, buf = len(table), C.cast(C.c_char_p(table), C.c_void_p)
        elif isinstance(table, (bytearray, memoryview)):
            table = bytes(table)
            n, buf = len(table), C.cast(C.c_char_p(table), C.c_void_p)
        elif isinstance(table, np.ndarray):
            n, buf = table.nbytes, table.ctypes.data_as(C.c_void_p)
        else:
            n, buf = int(length), C.c_void_p(int(table))
        bc, bh, failed, err = C.c_void_p(), C.c_void_p(), C.c_size_t(), _ErrStruct()
        rc = self._lib.L.amg_encode_changes(self.h, buf, C.c_size_t(n), C.byref(bc), C.byref(bh), C.byref(failed), C.byref(err))
        self._lib.check_indexed(rc, err, failed)
        hx = self._buffers(bh)[0].hex()
        return self._buffers(bc), [hx[i:i + 64] for i in range(0, len(hx), 64)]

    def last_encode_ms(self):
        """Device span of the last encode_flat call (CUDA events), ms."""
        return float(self._lib.L.amg_last_encode_ms(self.h))

    # ---- getHistory snapshots (src/automerge.js:105-118), on the device
    def history_patches_flat(self, lengths):
        """amg_get_history_patches: for every k in `lengths`, the FlatPatch of getPatch(loadChanges(init(), getAllChanges()[:k]))
        (k = 0 .. number of applied changes; repeats and any order allowed), filtered from the document's op table in one
        device call. The document is not touched."""
        lens = np.ascontiguousarray([int(k) for k in lengths], dtype=np.uint64)
        bl, err = C.c_void_p(), _ErrStruct()
        self._lib.check(self._lib.L.amg_get_history_patches(self.h, lens.ctypes.data_as(C.c_void_p), C.c_size_t(len(lens)), C.byref(bl), C.byref(err)), err)
        return [FlatPatch(raw) for raw in self._buffers(bl)]

    def history_patches(self, lengths):
        """history_patches_flat as patch dicts (what getPatch returns)."""
        return [fp.to_patch(True) for fp in self.history_patches_flat(lengths)]

    def last_history_ms(self):
        """Device span of the last history_patches_flat call (CUDA events), ms."""
        return float(self._lib.L.amg_last_history_ms(self.h))

    def dump_ops(self):
        rows, n, succ, m, err = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t(), _ErrStruct()
        self._lib.check(self._lib.L.amg_debug_dump_ops(self.h, C.byref(rows), C.byref(n), C.byref(succ), C.byref(m), C.byref(err)), err)
        r = np.frombuffer(C.string_at(rows, 8 * 8 * n.value), dtype=np.uint64).reshape(-1, 8).copy()
        s = np.frombuffer(C.string_at(succ, 8 * 2 * m.value), dtype=np.uint64).reshape(-1, 2).copy()
        self._lib.L.amg_free_mem(rows)
        self._lib.L.amg_free_mem(succ)
        return r, s

    def debug_decode(self, changes):
        """Decoded rows of a batch of binary changes straight from the decode kernels (amg_debug_decode): the document is
        not touched. Returns (hashes [n] bytes, n_ops [n], rows {column: uint32 array in batch order}, preds {'predActor',
        'predCtr'}, staged bytes that keyStrOff / valOff index: the changes back to back, DEFLATEd ones inflated)."""
        n = len(changes)
        blob = b''.join(bytes(c) for c in changes)
        offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum([len(c) for c in changes], out=offs[1:])
        buf = (C.c_uint8 * max(len(blob), 1)).from_buffer_copy(blob if blob else b'\0')
        hashes = (C.c_uint8 * (32 * max(n, 1)))()
        n_ops = np.zeros(max(n, 1), dtype=np.uint32)
        rows, total, total_preds, err = C.c_void_p(), C.c_size_t(), C.c_size_t(), _ErrStruct()
        self._lib.check(self._lib.L.amg_debug_decode(self.h, buf, offs.ctypes.data_as(C.c_void_p), C.c_size_t(n), hashes, n_ops.ctypes.data_as(C.c_void_p),
                                                     C.byref(rows), C.byref(total), C.byref(total_preds), C.byref(err)), err)
        M, P = total.value, total_preds.value
        flat = np.frombuffer(C.string_at(rows, 4 * (12 * M + 2 * P)), dtype=np.uint32).copy()
        self._lib.L.amg_free_mem(rows)
        names = ['objActor', 'objCtr', 'keyActor', 'keyCtr', 'keyStrOff', 'keyStrLen', 'insert', 'action', 'valLen', 'valOff', 'predNum', 'predOff']
        cols = {name: flat[k * M:(k + 1) * M] for k, name in enumerate(names)}
        preds = {'predActor': flat[12 * M:12 * M + P], 'predCtr': flat[12 * M + P:12 * M + 2 * P]}
        hs = bytes(hashes)
        return [hs[32 * i:32 * i + 32] for i in range(n)], n_ops[:n].copy(), cols, preds

    def debug_decode_column(self, buf, kind, n, parallel):
        """One document column through the parallel (True) or serial decoder; (rc, values, message), rc 1 = declined."""
        out = np.zeros(max(n, 1), dtype=np.int64)
        err = _ErrStruct()
        raw = bytes(buf)
        b = (C.c_uint8 * max(len(raw), 1)).from_buffer_copy(raw if raw else b'\0')
        rc = self._lib.L.amg_debug_decode_column(self.h, b, C.c_size_t(len(raw)), C.c_int(kind), C.c_size_t(n), C.c_int(1 if parallel else 0),
                                                 out.ctypes.data_as(C.c_void_p), C.byref(err))
        return rc, out[:n].tolist(), err.msg.decode('utf-8', 'replace')

    def timings(self):
        out = (C.c_float * 24)()
        self._lib.L.amg_last_timings(self.h, out, 24)
        return list(out)

    def launches(self):
        return int(self._lib.L.amg_kernel_launches(self.h))


def split_containers(buf):
    """columnar.js:829-837 splitContainers: the chunks of a buffer that holds several containers back to back."""
    from .columnar import _Dec, MAGIC, DecodeError
    d, chunks, start = _Dec(buf), [], 0
    while not d.done:   # decodeContainerHeader(decoder, false), columnar.js:688-708
        if d.raw(4) != MAGIC:
            raise DecodeError('Data does not begin with magic bytes 85 6f 4a 83')
        d.raw(4)
        d.raw(1)
        d.raw(d.uleb())
        chunks.append(d.buf[start:d.off])
        start = d.off
    return chunks


_decoders = {}


def _decoder_for(doc_class):
    """The per-process document handle that decodeChange / decodeChanges run on (created on first use, on AMG_DEVICE)."""
    if doc_class not in _decoders:
        _decoders[doc_class] = doc_class()
    return _decoders[doc_class]


def decode_changes(binary_changes, doc_class=None):
    """columnar.js:843-857 decodeChanges: every buffer may hold several containers; change chunks (type 1 or 2) of the whole
    list are decoded in one device call, a document chunk (type 0) contributes its changes (load, then the history decoded on
    the device), other chunk types are skipped. The error of the first failing chunk in input order is raised."""
    from .columnar import DecodeError
    doc_class = doc_class or GpuBackendDoc
    pieces, split_error = [], None   # ('change', chunk) / ('doc', chunk) in input order
    for b in binary_changes:
        try:
            chunks = split_containers(bytes(b))
        except DecodeError as e:
            split_error = AmgError(1, str(e))
            break
        for chunk in chunks:
            if chunk[8] == 0:
                pieces.append(('doc', chunk))
            elif chunk[8] in (1, 2):
                pieces.append(('change', chunk))
    changes = [c for kind, c in pieces if kind == 'change']
    table, failed, change_error = None, None, None
    if changes:
        try:
            table = _decoder_for(doc_class).decode_changes_flat(changes).to_changes()
        except AmgError as e:
            failed, change_error = e.failed_index, e
    out, k = [], 0
    for kind, chunk in pieces:
        if kind == 'doc':
            out.extend(doc_class(chunk).decode_history_flat().to_changes())
            continue
        if k == failed:
            raise change_error
        if table is not None:   # (after a failure only the chunks in front of the failing one are walked: for their errors)
            out.append(table[k])
        k += 1
    if split_error is not None:
        raise split_error
    return out


def doc_class_for(library_path):
    """A GpuBackendDoc subclass bound to another build of libamgpu (tests only)."""
    lib = Library(library_path)
    return type('BoundBackendDoc', (GpuBackendDoc,), {'_library': lib})
