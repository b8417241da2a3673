"""Device tables that applyChanges sizes from a bound instead of an exact count, driven to the edge of the bound.

To save host round trips, several tables of the apply path are sized before their exact length is known; a kernel then
writes up to the true count. A bound that is too small makes the kernel write past its table, and on the device that
silently corrupts a neighbouring table of the same slab. These scenarios build inputs where a careless bound is exceeded:
changes waiting in the queue (their bytes lie before this call's part of the arena), other-actor tables of one byte per
entry, and DEFLATE streams whose inflated sizes add up to more than 2^32 bytes.

Each scenario runs call by call against the oracle (patch, pendingChanges, heads, clock, getMissingDeps), then compares
save(), getChanges([]) and the op table, and applies an ordinary C3 batch on top (a corrupted neighbour often shows only
in the next call). The scenarios run twice:
- without a GPU, one subprocess per scenario on the AddressSanitizer build of the serial emulation
  (tests/_emu/build_asan.sh), where a write past a table is reported even when the result happens to come out right;
- on the GPU (-m gpu), in-process on libamgpu.so.
"""
import hashlib
import os
import random
import subprocess
import sys
import time
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == '__main__':
    sys.path[:0] = [HERE, ROOT]

import parity_checks  # noqa: E402
import replay  # noqa: E402
from automerge_classic_b200 import columnar, tracegen  # noqa: E402
from automerge_classic_b200.engine import AmgError  # noqa: E402
from doc_fixtures import gpu_doc  # noqa: E402,F401

AMG_ERR_UNSUPPORTED = 4


def _actor(rnd):
    return '%032x' % rnd.getrandbits(128)


def _hash(rnd):
    return '%064x' % rnd.getrandbits(256)


def _change(actor, seq=1, start_op=1, deps=(), ops=()):
    """a plain (never DEFLATEd) binary change and its hash"""
    return columnar.encode_change_raw({'actor': actor, 'seq': seq, 'startOp': start_op, 'time': 0, 'message': '',
                                       'deps': list(deps), 'ops': list(ops)}, compress=False)


def _set(key, value, pred=()):
    return {'action': 'set', 'obj': '_root', 'key': key, 'value': value, 'pred': list(pred)}


def _c3(seed, n=400):
    return tracegen.generate('C3', n, 3, seed=seed).changes()


class _Pair:
    """the engine document and the oracle document, fed the same calls and compared after each"""

    def __init__(self, Doc, oracle_mod):
        self.g, self.o = Doc(), oracle_mod.OracleDoc()

    def apply(self, changes):
        eo = eg = None
        try:
            po = self.o.apply_changes(changes)
        except Exception as e:   # noqa: BLE001 (the oracle's error class differs from the engine's)
            eo = str(e)
        try:
            pg = self.g.apply_changes(changes)
        except AmgError as e:
            eg = str(e)
        assert (eo is None) == (eg is None), (eo, eg)
        if eo is None:
            for k in ('maxOp', 'clock', 'deps', 'pendingChanges'):
                assert pg[k] == po[k], (k, pg[k], po[k])
            d = replay.deep_equal(replay.decode(pg), replay.decode(po))
            assert d is None, d
        else:
            assert eo.partition(': ')[2] == eg, (eo, eg)
        self.state()
        return eg

    def state(self):
        g, o = self.g, self.o
        assert sorted(g.heads()) == sorted(o.heads())
        assert g.clock() == o.clock()
        assert g.get_missing_deps() == o.get_missing_deps()

    def final(self, seed):
        g, o = self.g, self.o
        assert g.save() == o.save()
        assert g.get_changes([]) == o.get_changes([])
        parity_checks._dump_equal(g, o)
        # an ordinary batch on top: a table the scenario overran may have been a neighbour of one this call reads
        self.apply(_c3(seed))
        assert g.save() == o.save()
        parity_checks._dump_equal(g, o)
        d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(o.get_patch()))
        assert d is None, d


# ---------------------------------------------------------------------------------------------------------- dependencies
# depIdx holds one entry per dependency of every batch entry: the changes of this call and the Bq changes waiting in the
# queue. The queued changes' bytes lie below this call's part of the arena, so a bound from this call's bytes alone
# ((cur - arenaLen0) / 32 + B + 1) misses their dependencies: 12 queued changes of 100 dependencies each need 1 200
# entries, while one new change of ~3.3 KB bounds them at ~110.
def _queued_deps(rnd, n, pool, missing_every):
    """n changes from new actors, 100 dependencies each: hashes of `pool`, and (every `missing_every`-th change) one
    hash nobody has"""
    out = []
    for i in range(n):
        deps = rnd.sample(pool, 100)
        if missing_every and i % missing_every == 0:
            deps[rnd.randrange(100)] = _hash(rnd)
        out.append(_change(_actor(rnd), deps=deps, ops=[_set('k', i)])[0])
    return out


def _dep_pool(rnd, n=120):
    changes = [_change(_actor(rnd), ops=[_set('p%d' % j, j)]) for j in range(n)]
    return [c for c, _ in changes], [h for _, h in changes]


def scenario_queued_deps(Doc, oracle_mod, seed=1):
    """12 calls of one change each, 100 missing dependencies per change: all wait. Then the 120 changes they depend on
    arrive; the half whose dependencies are all among them is applied, the rest keeps waiting."""
    rnd = random.Random(seed)
    pool, pool_hashes = _dep_pool(rnd)
    p = _Pair(Doc, oracle_mod)
    for ch in _queued_deps(rnd, 12, pool_hashes, 2):
        p.apply([ch])
    p.apply(pool)
    p.final(seed)


def scenario_queued_deps_with_batch(Doc, oracle_mod, seed=2):
    """A queue of changes with 100 dependencies each meets an ordinary C3 batch in one call, on a clone. A clone has the
    queue but none of the grown scratch tables, so the batch alone sizes them: the 30 queued changes need 3 000 entries
    next to the batch's ~100, and the batch's 11 KB bound them at ~480."""
    rnd = random.Random(seed)
    pool, pool_hashes = _dep_pool(rnd)
    p = _Pair(Doc, oracle_mod)
    p.apply(_queued_deps(rnd, 30, pool_hashes, 3))
    p.g, p.o = p.g.clone(), p.o.clone()
    p.apply(_c3(seed + 100, 100))
    p.apply(pool[:60])
    p.apply(pool[60:] + _c3(seed + 200, 200))
    p.final(seed)


# ---------------------------------------------------------------------------------------------------------- actor tables
# amap holds, for every change this call applies, its author and one entry per other-actor table entry. The bound
# B + (cur - arenaLen0) / 2 + 2 assumed two bytes per entry of this call's bytes. Changes released from the queue are
# applied too, but their bytes are not in that range: 50 queued changes naming 30 other actors each need
# 1 + 50 * 31 = 1 551 entries when the ~60-byte change they wait for arrives, and the bound gives 51 + 30 + 2 = 83.
def _actor_tables(rnd):
    actors = [_actor(rnd) for _ in range(30)]
    first = [_change(a, ops=[_set('k', i)])[0] for i, a in enumerate(actors)]
    held, held_hash = _change(_actor(rnd), ops=[_set('m', 1)])
    pred = ['1@%s' % a for a in actors]
    waiting = [_change(_actor(rnd), start_op=2, deps=[held_hash], ops=[_set('k', 100 + i, pred)])[0] for i in range(50)]
    return first, held, waiting


def scenario_queued_actor_tables(Doc, oracle_mod, seed=3):
    rnd = random.Random(seed)
    first, held, waiting = _actor_tables(rnd)
    p = _Pair(Doc, oracle_mod)
    p.apply(first)
    p.apply(waiting)
    p.apply([held])
    p.final(seed)


def scenario_queued_actor_tables_one_by_one(Doc, oracle_mod, seed=4):
    """the 50 waiting changes arrive in 50 calls before the change they wait for"""
    rnd = random.Random(seed)
    first, held, waiting = _actor_tables(rnd)
    p = _Pair(Doc, oracle_mod)
    p.apply(first)
    for ch in waiting:
        p.apply([ch])
    p.apply([held])
    p.final(seed)


def _with_other_actors(change, others):
    """`change` (plain, no deps, no other actors, seq / startOp / time below 128, no message) with `others` as its
    other-actor table; checksum recomputed"""
    raw = bytes(change)
    assert raw[8] == 1
    r = 9
    while raw[r] & 0x80:   # body length
        r += 1
    body = bytearray(raw[r + 1:])
    assert body[0] == 0   # no deps
    pos = 2 + body[1]     # author: length-prefixed
    pos += 3              # seq, startOp, time: one byte each
    assert body[pos] == 0   # empty message
    pos += 1
    assert body[pos] == 0   # no other actors
    body[pos:pos + 1] = columnar.uleb(len(others)) + b''.join(columnar.prefixed(a) for a in others)
    header = bytes([1]) + columnar.uleb(len(body))
    digest = hashlib.sha256(header + bytes(body)).digest()
    return columnar.MAGIC + digest[:4] + header + bytes(body)


def scenario_empty_actor_ids(Doc, oracle_mod, seed=5):
    """A change whose other-actor table holds 1 000 empty actor ids: one byte each, so a bound of one entry per two bytes
    is exceeded by the change alone. The author is known, the empty ids are not."""
    rnd = random.Random(seed)
    p = _Pair(Doc, oracle_mod)
    author = _actor(rnd)
    p.apply([_change(author, ops=[_set('a', 1)])[0]])
    ch = _with_other_actors(_change(author, seq=2, start_op=2, deps=(), ops=[_set('b', 2)])[0], [b''] * 1000)
    p.apply([ch])
    p.final(seed)


# ---------------------------------------------------------------------------------------------------------- inflate
# A DEFLATEd change may inflate to almost 2^31 bytes (KE_TOO_LARGE above that). The inflated sizes are laid out behind the
# batch by a prefix sum; two streams of 2^31 - 1 body bytes each add up to 2^32 + 26, which wraps to 26 in 32 bits. The
# total has to be taken in 64 bits, and the call refused with "change arena limited to 4 GiB" before anything is placed.
_BIG = {}


def _big_stream(body_len):
    """a chunk of type 2 whose body inflates to body_len bytes: a valid change header with a message of zeros. Built
    in pieces, so that the host never holds the inflated body: after a full flush the compressor starts afresh, so every
    4 MiB block of zeros compresses to the same bytes and is compressed once."""
    if body_len in _BIG:
        return _BIG[body_len]
    actor = bytes(range(1, 17))
    head = b'\x00' + columnar.prefixed(actor) + b'\x01\x01\x00'
    tail = b'\x00\x00'   # no other actors, no columns
    msg_len = body_len - len(head) - len(tail)
    msg_len -= len(columnar.uleb(msg_len))
    head += columnar.uleb(msg_len)
    assert len(head) + msg_len + len(tail) == body_len
    sha = hashlib.sha256(bytes([1]) + columnar.uleb(body_len))
    co = zlib.compressobj(9, zlib.DEFLATED, -15)
    parts = [co.compress(head) + co.flush(zlib.Z_FULL_FLUSH)]
    sha.update(head)
    block = bytes(1 << 22)
    whole, rest = divmod(msg_len, len(block))
    packed = co.compress(block) + co.flush(zlib.Z_FULL_FLUSH)
    for _ in range(whole):
        sha.update(block)
        parts.append(packed)
    sha.update(block[:rest])
    sha.update(tail)
    parts.append(co.compress(block[:rest]) + co.compress(tail) + co.flush())
    comp = b''.join(parts)
    out = columnar.MAGIC + sha.digest()[:4] + bytes([2]) + columnar.uleb(len(comp)) + comp
    _BIG[body_len] = out
    return out


def _expect_arena_limit(fn, what):
    t0 = time.time()
    with pytest.raises(AmgError) as ei:
        fn()
    assert ei.value.code == AMG_ERR_UNSUPPORTED, (what, ei.value.code, str(ei.value))
    assert 'change arena limited to 4 GiB' in str(ei.value), (what, str(ei.value))
    print('%s: refused in %.2f s' % (what, time.time() - t0))


def scenario_inflated_past_4gib(Doc, oracle_mod, seed=6):
    """two and three streams of 2^31 - 1 body bytes, through applyChanges and decodeChanges: refused, document untouched"""
    big = _big_stream((1 << 31) - 1)
    base = _c3(seed, 600)
    p = _Pair(Doc, oracle_mod)
    p.apply(base[:300])
    saved = p.g.save()
    for k in (2, 3):
        batch = [base[300]] + [big] * k
        _expect_arena_limit(lambda: p.g.apply_changes(batch), 'applyChanges, %d streams' % k)
        assert p.g.save() == saved
        p.state()
        blob = b''.join(batch)
        offs = np.zeros(len(batch) + 1, dtype=np.uint64)
        np.cumsum([len(c) for c in batch], out=offs[1:])
        _expect_arena_limit(lambda: p.g.decode_packed_flat(blob, offs, len(batch)), 'decodeChanges, %d streams' % k)
    p.apply(base[300:])
    p.final(seed)


SCENARIOS = {f.__name__[len('scenario_'):]: f for f in (
    scenario_queued_deps, scenario_queued_deps_with_batch, scenario_queued_actor_tables,
    scenario_queued_actor_tables_one_by_one, scenario_empty_actor_ids, scenario_inflated_past_4gib)}


# ---------------------------------------------------------------------------------------------------------- CPU: ASAN
def _asan_runtime():
    try:
        out = subprocess.run(['gcc', '-print-file-name=libasan.so'], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None
    return out if os.path.isabs(out) and os.path.exists(out) else None


@pytest.fixture(scope='module')
def asan_lib(oracle_mod):
    asan = _asan_runtime()
    if asan is None:
        pytest.skip('no AddressSanitizer runtime: gcc -print-file-name=libasan.so finds no libasan.so')
    lib = os.path.join(HERE, '_emu', 'libamgpu_emu_asan.so')
    src = os.path.join(ROOT, 'automerge_classic_b200', 'csrc')
    newest = max(os.path.getmtime(os.path.join(src, f)) for f in os.listdir(src))
    if not os.path.exists(lib) or os.path.getmtime(lib) < newest:   # (the instrumented build takes minutes)
        subprocess.check_call([os.path.join(HERE, '_emu', 'build_asan.sh')])
    from automerge_classic_b200 import build
    build.build_tracegen()
    stdcxx = subprocess.run(['gcc', '-print-file-name=libstdc++.so.6'], capture_output=True, text=True).stdout.strip()
    return asan, stdcxx


@pytest.mark.parametrize('name', sorted(SCENARIOS))
def test_sizing_bounds_asan(asan_lib, name):
    asan, stdcxx = asan_lib
    env = dict(os.environ, LD_PRELOAD='%s %s' % (asan, stdcxx), ASAN_OPTIONS='detect_leaks=0')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + [os.path.abspath(__file__), name], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    report = [ln for ln in r.stderr.splitlines() if 'AddressSanitizer' in ln or 'runtime error' in ln]
    assert r.returncode == 0 and not report, '%s: exit %d\n%s\n%s' % (name, r.returncode, r.stdout[-3000:], r.stderr[-6000:])


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(SCENARIOS))
def test_sizing_bounds_gpu(gpu_doc, oracle_mod, name):   # noqa: F811
    SCENARIOS[name](gpu_doc, oracle_mod)


if __name__ == '__main__':
    import oracle
    from automerge_classic_b200.engine import doc_class_for
    SCENARIOS[sys.argv[1]](doc_class_for(os.path.join(HERE, '_emu', 'libamgpu_emu_asan.so')), oracle)
    print('ok', sys.argv[1])
