"""applyLocalChange on the device (GpuBackendDoc.apply_local_change, Engine::applyLocalChange): the change request is
encoded with the author's previous change hash added to its deps and applied from device memory. Every scenario runs the
device route, the host route (the same document class with the device route switched off) and the oracle through
Backend.applyLocalChange, and compares them. CPU run on the serial emulation build, GPU run on libamgpu.so."""
import random

import pytest

import replay
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401

LOCAL = 'a1' * 16
REMOTES = ('b2' * 16, 'c3' * 8)


def host_route(Doc):
    """Doc with the device route switched off: Backend.applyLocalChange then encodes on the host and applies the bytes"""
    return type('HostRoute' + Doc.__name__, (Doc,), {'apply_local_change': None})


def _trace(cfg, n, a, seed=0):
    from automerge_classic_b200 import tracegen
    return tracegen.generate(cfg, n, a, seed=seed).changes()


def _hash(change):
    from automerge_classic_b200 import columnar
    return columnar.decode_change(bytes(change))['hash']


def _state(doc):
    fp = doc._state()
    return fp.deps, fp.clock, fp.max_op, fp.pending


class Session:
    """One document three times: device route, host route, oracle. Starts from `changes` applied, or from load(save(them))."""

    def __init__(self, Doc, oracle_mod, changes=(), load=False):
        from automerge_classic_b200.backend import Backend
        self.Doc, self.H = Doc, host_route(Doc)
        self.B = [Backend(Doc), Backend(self.H), Backend(oracle_mod.OracleDoc)]
        self.h = []
        for cls, B in zip((Doc, self.H, oracle_mod.OracleDoc), self.B):
            s = B.init()
            if changes:
                s = B.applyChanges(s, list(changes))[0]
            if load:
                s = B.load(B.save(s))
            self.h.append(s)
        self.new_hashes = []

    @property
    def dev(self):
        return self.h[0]['state']

    @property
    def host(self):
        return self.h[1]['state']

    def local(self, change, what):
        out = []
        for i, B in enumerate(self.B):
            self.h[i], patch, binary = B.applyLocalChange(self.h[i], dict(change))
            out.append((patch, bytes(binary)))
        (pd, bd), (ph, bh), (po, bo) = out
        assert bd == bh == bo, what
        assert pd == ph, what
        d = replay.deep_equal(replay.decode(pd), replay.decode(po))
        assert d is None, (what, d)
        assert _state(self.dev) == _state(self.host), what
        self.new_hashes.append(_hash(bd))
        return pd, bd

    def remote(self, changes, what):
        ps = [B.applyChanges(self.h[i], list(changes)) for i, B in enumerate(self.B)]
        for i in range(3):
            self.h[i] = ps[i][0]
        assert ps[0][1] == ps[1][1], what
        assert replay.deep_equal(replay.decode(ps[0][1]), replay.decode(ps[2][1])) is None, what

    def check_exports(self, what, peer=None):
        dev, host, orc = (h['state'] for h in self.h)
        assert dev.save() == host.save() == orc.save(), what
        assert dev.get_patch_flat().raw == host.get_patch_flat().raw, what
        all_dev = [bytes(c) for c in dev.get_changes([])]
        assert all_dev == [bytes(c) for c in host.get_changes([])] == [bytes(c) for c in orc.get_changes([])], what
        for h in self.new_hashes:
            assert bytes(dev.get_change_by_hash(h)) == bytes(host.get_change_by_hash(h)), what
        if peer is not None:
            p = self.Doc()
            p.apply_changes(list(peer), want_patch=False)
            assert [bytes(c) for c in dev.get_changes_added(p)] == [bytes(c) for c in host.get_changes_added(p)], what
            assert [bytes(c) for c in p.get_changes_added(dev)] == [bytes(c) for c in p.get_changes_added(host)], what

    def request(self, actor, ops, deps=None, **extra):
        seq = self.dev.clock_of(actor) + 1
        ch = {'actor': actor, 'seq': seq, 'startOp': self.dev.max_op() + 1, 'time': 0,
              'deps': list(self.dev.heads()) if deps is None else deps, 'ops': ops}
        ch.update(extra)
        return ch


def _values(rnd, n):
    dt = rnd.choice((None, 'int', 'uint', 'counter', 'timestamp', 'float64'))
    if dt is None:
        return [rnd.choice(('a', 'ünï', True, None, 'x' * 9)) for _ in range(n)], None
    if dt == 'float64':
        return [float(rnd.randrange(-9, 9)) for _ in range(n)], dt
    return [rnd.randrange(0 if dt == 'uint' else -50, 50) for _ in range(n)], dt


def edit_ops(rnd, s, model, actor, start, big=False):
    """Ops of one local edit that applies to the document `model` describes (model is updated)"""
    ops, op = [], start
    def add(o):
        nonlocal op
        ops.append(o)
        first = op
        op += len(o['values']) if 'values' in o else o.get('multiOp', 1)
        return first
    kind = rnd.randrange(6) if not big else 1
    if model.get('list') is None:
        model['list'] = '%d@%s' % (add({'action': 'makeList', 'obj': '_root', 'key': 'list', 'pred': []}), actor)
        model['elems'] = []
    if kind == 0:   # map keys with every kind of value, unicode keys
        for key in rnd.sample(['a', 'b', 'ключ', 'bird🐦', 'x' * 20], 2):
            v, dt = _values(rnd, 1)
            o = {'action': 'set', 'obj': '_root', 'key': key, 'value': v[0], 'pred': model['keys'].get(key, [])}
            if dt:
                o['datatype'] = dt
            model['keys'][key] = ['%d@%s' % (add(o), actor)]
    elif kind == 1:   # multi-insert values
        v, dt = _values(rnd, 60 if big else rnd.randrange(1, 6))
        if big:
            v, dt = ['text %d' % i for i in range(len(v))], None
        ref = model['elems'][-1] if model['elems'] and rnd.random() < 0.5 else '_head'
        o = {'action': 'set', 'obj': model['list'], 'elemId': ref, 'insert': True, 'values': v, 'pred': []}
        if dt:
            o['datatype'] = dt
        first = add(o)
        model['runs'].append((first, len(v)))
        model['elems'] += ['%d@%s' % (first + i, actor) for i in range(len(v))]
    elif kind == 2 and model['runs']:   # multiOp delete of the start of a run
        first, n = model['runs'].pop()
        k = rnd.randrange(1, n + 1)
        e = '%d@%s' % (first, actor)
        o = {'action': 'del', 'obj': model['list'], 'elemId': e, 'pred': [e]}
        if k > 1:
            o['multiOp'] = k
        add(o)
        gone = {'%d@%s' % (first + i, actor) for i in range(k)}
        model['elems'] = [x for x in model['elems'] if x not in gone]
    elif kind == 3:   # objects
        for act in rnd.sample(['makeMap', 'makeText', 'makeTable', 'makeList'], 2):
            key = 'obj-' + act
            model['keys'][key] = ['%d@%s' % (add({'action': act, 'obj': '_root', 'key': key, 'pred': model['keys'].get(key, [])}), actor)]
    elif kind == 4:   # counter and inc
        if model.get('counter') is None:
            model['counter'] = '%d@%s' % (add({'action': 'set', 'obj': '_root', 'key': 'cnt', 'value': 5, 'datatype': 'counter', 'pred': model['keys'].get('cnt', [])}), actor)
            model['keys']['cnt'] = [model['counter']]
        else:
            model['keys']['cnt'] = ['%d@%s' % (add({'action': 'inc', 'obj': '_root', 'key': 'cnt', 'value': rnd.randrange(1, 9), 'pred': [model['counter']]}), actor)]
    else:   # a key set and deleted
        k = '%d@%s' % (add({'action': 'set', 'obj': '_root', 'key': 'tmp', 'value': 't', 'pred': model['keys'].get('tmp', [])}), actor)
        add({'action': 'del', 'obj': '_root', 'key': 'tmp', 'pred': [k]})
        model['keys']['tmp'] = []
    return ops


def new_model():
    return {'keys': {}, 'runs': [], 'list': None, 'elems': []}


def edits(S, rnd, model, n, what, actor=LOCAL):
    for i in range(n):
        ops = edit_ops(rnd, S, model, actor, S.dev.max_op() + 1)
        extra = {}
        if rnd.random() < 0.5:
            extra['message'] = rnd.choice(('', 'edit', 'ünïcødé ✓'))
        if rnd.random() < 0.5:
            extra['time'] = rnd.randrange(0, 2 ** 40)
        S.local(S.request(actor, ops, **extra), (what, i))


def check_chain(Doc, oracle_mod):
    """The first change of a new actor, a chain of edits of every op kind, deps that repeat or hold the previous hash"""
    rnd = random.Random(1)
    S = Session(Doc, oracle_mod)
    model = new_model()
    edits(S, rnd, model, 25, 'chain')
    prev = S.new_hashes[-1]
    heads = S.dev.heads()
    # deps already holding the previous hash, unsorted and repeated deps, and no deps at all
    for deps in ([prev], heads[::-1] + heads, [], [prev, prev]):
        S.local(S.request(LOCAL, edit_ops(rnd, S, model, LOCAL, S.dev.max_op() + 1), deps=list(deps)), ('deps', len(deps)))
    S.check_exports('chain')


def check_large(Doc, oracle_mod):
    """A change of 256 bytes or more comes back DEFLATEd and goes out DEFLATEd afterwards"""
    rnd = random.Random(2)
    S = Session(Doc, oracle_mod, _trace('C8', 200, 3))
    model = new_model()
    for i in range(3):
        _, binary = S.local(S.request(LOCAL, edit_ops(rnd, S, model, LOCAL, S.dev.max_op() + 1, big=True)), ('large', i))
        assert binary[8] == 2, i
    S.check_exports('large', peer=_trace('C8', 200, 3)[:50])


def check_interleaved(Doc, oracle_mod):
    """Local edits between remote changes of two other actors, then a clone that carries on"""
    rnd = random.Random(3)
    base = _trace('C3', 300, 4)
    S = Session(Doc, oracle_mod, base[:100])
    model = new_model()
    rest = base[100:]
    for i in range(8):
        edits(S, rnd, model, 2, ('interleaved', i))
        S.remote(rest[25 * i:25 * (i + 1)], ('remote', i))
    # remote changes of two other actors, made on a peer that had the local edits
    from automerge_classic_b200.backend import Backend
    P = Backend(Doc)
    p = P.applyChanges(P.init(), [bytes(c) for c in S.dev.get_changes([])])[0]
    remote = []
    for j, actor in enumerate(REMOTES * 2):
        ops = [{'action': 'set', 'obj': '_root', 'key': 'r%d' % j, 'value': j, 'pred': []}]
        ch = {'actor': actor, 'seq': p['state'].clock_of(actor) + 1, 'startOp': p['state'].max_op() + 1, 'time': 0, 'deps': [], 'ops': ops}
        p, _, b = P.applyLocalChange(p, ch)
        remote.append(b)
    S.remote(remote, 'two actors')
    edits(S, rnd, model, 3, 'after two actors')
    S.check_exports('interleaved', peer=base[:150])
    # clones carry on from the same last change
    for i in range(3):
        S.h = [{'state': h['state'].clone(), 'heads': h['heads']} for h in S.h]
        edits(S, rnd, model, 2, ('clone', i))
    S.check_exports('clones')


def check_queued(Doc, oracle_mod):
    """A local change that makes queued changes ready: the same request made first on a replica, a peer builds on it"""
    from automerge_classic_b200.backend import Backend
    rnd = random.Random(4)
    base = _trace('C6', 200, 3)
    S = Session(Doc, oracle_mod, base)
    model = new_model()
    edits(S, rnd, model, 2, 'before')
    req = S.request(LOCAL, edit_ops(rnd, S, model, LOCAL, S.dev.max_op() + 1))
    B = Backend(Doc)
    r = B.applyChanges(B.init(), [bytes(c) for c in S.dev.get_changes([])])[0]
    r, _, first = B.applyLocalChange(r, dict(req))
    ch = {'actor': REMOTES[0], 'seq': 1, 'startOp': r['state'].max_op() + 1, 'time': 0, 'deps': [_hash(first)],
          'ops': [{'action': 'set', 'obj': '_root', 'key': 'after', 'value': 1, 'pred': []}]}
    r, _, waiting = B.applyLocalChange(r, ch)
    S.remote([waiting], 'queued')
    assert _state(S.dev)[3] == 1
    S.local(req, 'makes the queue ready')
    assert _state(S.dev)[3] == 0
    edits(S, rnd, model, 2, 'after')
    S.check_exports('queued')


def _loaded_cases(Doc, oracle_mod, base, rnd):
    """(what, changes, model, local actor's last change is a head) of documents to load: the local actor's last change the
    single head; another actor's change on top of it the single head; two other actors' changes on top of it; the local
    actor's change and another actor's concurrent change both heads"""
    def session(extra_actors, concurrent):
        S = Session(Doc, oracle_mod, base)
        model = new_model()
        edits(S, rnd, model, 2, 'pre-load')
        before_last = S.dev.heads()
        edits(S, rnd, model, 1, 'pre-load, last')
        deps = before_last if concurrent else S.dev.heads()
        for j, actor in enumerate(extra_actors):
            ops = [{'action': 'set', 'obj': '_root', 'key': 'on-top-%d' % j, 'value': j, 'pred': []}]
            S.local(S.request(actor, ops, deps=list(deps)), ('on top', actor))
        return [bytes(c) for c in S.dev.get_changes([])], model, S.new_hashes[2]
    out = []
    for what, extra, concurrent in (('own head', (), False), ('other head', REMOTES[:1], False),
                                    ('several other heads', REMOTES, False), ('own and other head', REMOTES[:1], True)):
        changes, model, mine = session(extra, concurrent)
        out.append((what, changes, model, mine))
    return out


def _alternating(n, actors=('d4' * 16, 'e5' * 16, 'f6' * 8)):
    """n single-op changes whose authors take turns, each depending on the one before"""
    from automerge_classic_b200.columnar import encode_change
    out, last, seq, pred = [], [], {a: 0 for a in actors}, {}
    for i in range(n):
        a, key = actors[i % len(actors)], 'k%d' % (i % 40)
        seq[a] += 1
        ch = encode_change({'actor': a, 'seq': seq[a], 'startOp': i + 1, 'time': 0, 'deps': last,
                            'ops': [{'action': 'set', 'obj': '_root', 'key': key, 'value': i, 'pred': pred.get(key, [])}]})
        pred[key] = ['%d@%s' % (i + 1, a)]
        last = [_hash(ch)]
        out.append(ch)
    return out


def check_loaded(Doc, oracle_mod, base=None):
    """After load: the local actor's last change the single head; another actor's change the head (the history is rebuilt
    for the previous hash); several heads with and without the local actor's change among them"""
    rnd = random.Random(5)
    base = base or _trace('C3', 200, 3)
    for what, changes, model, mine in _loaded_cases(Doc, oracle_mod, base, rnd):
        S = Session(Doc, oracle_mod, changes, load=True)
        heads = S.dev.heads()
        assert (mine in heads) == (what in ('own head', 'own and other head')), (what, heads)
        assert len(heads) == (2 if what in ('several other heads', 'own and other head') else 1), (what, heads)
        edits(S, rnd, model, 4, what)
        S.check_exports(what)


def check_loaded_long(Doc, oracle_mod):
    """The same on 5 000 changes whose authors take turns: a change metadata column long enough that the load checks the
    clock, and finds each actor's last change, on the device (ClockCheckKernel)"""
    check_loaded(Doc, oracle_mod, _alternating(5000))


def check_traces(Doc, oracle_mod):
    """Trace prefixes with local edits on top, also by an actor of the trace"""
    rnd = random.Random(6)
    for cfg, n, a in (('C3', 400, 4), ('C4', 1200, 3), ('C8', 300, 3)):
        ch = _trace(cfg, n, a)
        S = Session(Doc, oracle_mod, ch[:len(ch) * 2 // 3])
        model = new_model()
        edits(S, rnd, model, 4, cfg)
        S.remote(ch[len(ch) * 2 // 3:], (cfg, 'rest'))
        edits(S, rnd, model, 2, (cfg, 'after rest'))
        for i, trace_actor in enumerate(sorted(S.dev.clock())[:2]):
            ops = [{'action': 'set', 'obj': '_root', 'key': 'by-trace-actor', 'value': i, 'pred': []}]
            S.local(S.request(trace_actor, ops), (cfg, 'trace actor', i))
        S.check_exports(cfg)


def _error(call):
    try:
        call()
    except Exception as e:   # noqa: BLE001
        return type(e), str(e)
    return None


def check_errors(Doc, oracle_mod):
    """Each error as the host route raises it; the document unchanged afterwards, and the next valid call goes through"""
    from automerge_classic_b200.engine import AmgError, FlatChanges
    rnd = random.Random(7)
    S = Session(Doc, oracle_mod, _trace('C3', 100, 3))
    model = new_model()
    edits(S, rnd, model, 3, 'setup')
    seq, start, heads = S.dev.clock_of(LOCAL), S.dev.max_op() + 1, S.dev.heads()
    good = [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': []}]
    bad_dict = [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': ['not an op id']}]
    other = REMOTES[0]

    def req(**kw):
        ch = {'actor': LOCAL, 'seq': seq + 1, 'startOp': start, 'time': 0, 'deps': heads, 'ops': good}
        ch.update(kw)
        return ch
    cases = [
        ('already applied', req(seq=seq)),
        ('skipped', req(seq=seq + 2)),
        ('already applied, malformed', req(seq=seq, ops=bad_dict)),
        ('skipped, malformed', req(seq=seq + 2, ops=bad_dict)),
        ('no matching pred', req(ops=[{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': ['999@' + LOCAL]}])),
        ('unknown object', req(ops=[{'action': 'set', 'obj': '77@' + LOCAL, 'key': 'k', 'value': 1, 'pred': []}])),
        ('missing reference element', req(ops=[{'action': 'set', 'obj': model['list'], 'elemId': '555@' + LOCAL, 'insert': True, 'value': 1, 'pred': []}])),
        ('unknown actor in a pred', req(ops=[{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': ['1@' + other]}])),
        ('counter beyond 32 bits', req(ops=[{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': ['%d@%s' % (2 ** 32 + 5, LOCAL)]}])),
    ]
    for what, ch in cases:
        before = [(h['state'].save(), h['state'].get_patch_flat().raw) for h in S.h[:2]]
        handles = [dict(h) for h in S.h]
        got = [_error(lambda: B.applyLocalChange(handles[i], dict(ch))) for i, B in enumerate(S.B[:2])]
        assert got[0] is not None and got[0] == got[1], (what, got)
        assert [(h['state'].save(), h['state'].get_patch_flat().raw) for h in S.h[:2]] == before, what
    # an encoder-level error: the message of the host codec (which raises it as a ValueError), as a RangeError, and the
    # error encodeChange raises on the device for the same request
    ch = req(time=2 ** 60)
    before = (S.dev.save(), S.dev.get_patch_flat().raw)
    with pytest.raises(AmgError) as dev_err:
        S.B[0].applyLocalChange(dict(S.h[0]), dict(ch))
    with pytest.raises(ValueError) as host_err:
        S.B[1].applyLocalChange(dict(S.h[1]), dict(ch))
    assert (dev_err.value.kind, str(dev_err.value)) == ('RangeError', str(host_err.value)), (dev_err.value, host_err.value)
    assert _error(lambda: Doc().encode_flat(FlatChanges.from_changes([dict(ch, deps=sorted(set(heads + [S.new_hashes[-1]])))]))) == (AmgError, str(dev_err.value))
    assert (S.dev.save(), S.dev.get_patch_flat().raw) == before
    # the next valid call succeeds on every route
    S.local(req(), 'after the errors')
    S.check_exports('errors')


def check_waiting(Doc, oracle_mod):
    """A local change whose deps are not all applied waits in the queue; the call then raises the reference's RangeError
    "Unknown change" with the handle frozen, on every route. Once the missing change arrives, the queue applies it."""
    from automerge_classic_b200.backend import Backend, RangeError
    rnd = random.Random(8)
    S = Session(Doc, oracle_mod, _trace('C8', 150, 3))
    model = new_model()
    edits(S, rnd, model, 2, 'before')
    B = Backend(Doc)
    r = B.applyChanges(B.init(), [bytes(c) for c in S.dev.get_changes([])])[0]
    missing = []   # one change per round that the document has not seen
    for actor in REMOTES:
        ch = {'actor': actor, 'seq': 1, 'startOp': r['state'].max_op() + 1, 'time': 0, 'deps': r['state'].heads(),
              'ops': [{'action': 'set', 'obj': '_root', 'key': 'missing-' + actor, 'value': 1, 'pred': []}]}
        r, _, m = B.applyLocalChange(r, ch)
        missing.append(m)
    for big, missing in zip((False, True), missing):   # the waiting change plain, and one of 256 bytes or more
        ops = edit_ops(rnd, S, model, LOCAL, S.dev.max_op() + 1, big=big)
        req = S.request(LOCAL, ops, deps=S.dev.heads() + [_hash(missing)])
        errors = []
        for i, B in enumerate(S.B):
            with pytest.raises(RangeError) as e:
                B.applyLocalChange(S.h[i], dict(req))
            assert S.h[i]['frozen'], i
            errors.append(str(e.value))
            S.h[i] = {'state': S.h[i]['state'], 'heads': S.h[i]['state'].heads()}
        assert errors == ['Unknown change: actorId = %s, seq = %d' % (LOCAL, req['seq'])] * 3, errors
        assert _state(S.dev) == _state(S.host) and _state(S.dev)[3] == 1
        assert S.dev.save() == S.host.save()
        if not big:
            S.remote([missing], 'the missing change')
            assert _state(S.dev) == _state(S.host) and _state(S.dev)[3] == 0
            edits(S, rnd, model, 2, 'after')
    S.check_exports('waiting')


def check_abi(Doc, oracle_mod):
    """apply_local_change_flat: the patch without the new hash in its deps, want_patch=False, a table of two changes"""
    from automerge_classic_b200.engine import AmgError, FlatChanges
    d = Doc()
    ch = {'actor': LOCAL, 'seq': 1, 'startOp': 1, 'time': 0, 'deps': [], 'ops': [{'action': 'set', 'obj': '_root', 'key': 'a', 'value': 1, 'pred': []}]}
    fp, b1 = d.apply_local_change_flat(ch)
    assert fp.deps == [] and d.heads() == [_hash(b1)]
    ch2 = dict(ch, seq=2, startOp=2)
    assert d.apply_local_change_flat(ch2, want_patch=False)[0] is None
    assert d.clock() == {LOCAL: 2}
    table = FlatChanges.from_changes([dict(ch, seq=3, startOp=3), dict(ch, seq=4, startOp=4)]).raw
    import ctypes as C
    pp, bl = C.c_void_p(), C.c_void_p()
    from automerge_classic_b200.engine import _ErrStruct
    err = _ErrStruct()
    rc = d._lib.L.amg_apply_local_change(d.h, C.cast(C.c_char_p(table), C.c_void_p), C.c_size_t(len(table)), 1, C.byref(pp), C.byref(bl), C.byref(err))
    assert rc == 1 and b'one change request' in err.msg
    with pytest.raises(AmgError, match='already been applied'):
        d.apply_local_change_flat(ch2)
    assert d.clock() == {LOCAL: 2}


ALL = (check_chain, check_large, check_interleaved, check_queued, check_loaded, check_loaded_long, check_traces, check_errors, check_waiting,
       check_abi)


@pytest.mark.parametrize('check', ALL, ids=[c.__name__ for c in ALL])
def test_local_change_emu(emu_doc, oracle_mod, check):
    check(emu_doc, oracle_mod)


@pytest.mark.gpu
@pytest.mark.parametrize('check', ALL, ids=[c.__name__ for c in ALL])
def test_local_change_gpu(gpu_doc, oracle_mod, check):
    check(gpu_doc, oracle_mod)


@pytest.mark.gpu
def test_span_gpu(gpu_doc):
    """the call times itself into its own span and no other"""
    d = gpu_doc()
    d.sync_bloom([])
    spans = {k: getattr(d, 'last_%s_ms' % k)() for k in ('sync', 'decode', 'encode', 'history', 'merge')}
    ch = {'actor': LOCAL, 'seq': 1, 'startOp': 1, 'time': 0, 'deps': [], 'ops': [{'action': 'set', 'obj': '_root', 'key': 'a', 'value': 1, 'pred': []}]}
    d.apply_local_change_flat(ch)
    assert d.last_local_ms() > 0
    assert {k: getattr(d, 'last_%s_ms' % k)() for k in spans} == spans
