"""What the device entry points share (csrc/engine_impl.cuh): the device span behind amg_last_*_ms, the error word, the
dependency lookup over change headers and the failing-change search. On the emulation build, one call of each entry point
launches a pinned number of kernels; on the H100, each call kind times itself into its own span."""
import random

import pytest

from doc_fixtures import emu_doc, gpu_doc  # noqa: F401
from test_decode_changes import _deflate

SPANS = ('sync', 'decode', 'encode', 'history', 'merge')

# Kernel launches of one call of each entry point on the inputs of _entry_point_calls, measured on the emulation build
# before the entry points shared their plumbing. Sharing it must not add, drop or reorder a launch.
EXPECTED_LAUNCHES = {'sync_bloom_all': 1, 'sync_bloom_last_sync': 1, 'sync_changes_to_send': 7, 'decode_changes': 21, 'decode_history': 12,
                     'encode': 138, 'history_patches': 144, 'merge': 225, 'save': 256}


def _trace():
    from automerge_classic_b200 import tracegen
    return tracegen.generate('C3', 300, 4, seed=0).changes()


def _doc(Doc, changes):
    d = Doc()
    d.apply_changes(changes, want_patch=False)
    return d


def _entry_point_calls(Doc):
    """(name, document, call) for one call of each entry point, in the order they run"""
    from automerge_classic_b200 import sync
    ch = _trace()
    d = _doc(Doc, ch)
    hashes = [sync._change_meta(c)['hash'] for c in ch]
    rnd = random.Random(0)
    mixed = [_deflate(c, 6) if rnd.random() < 0.5 else c for c in ch[:120]]
    table = d.decode_changes_flat(ch[:80])
    remote = Doc(d.save())                      # loaded: merging from it rebuilds its history first
    local = _doc(Doc, ch[:150])
    later = Doc(_doc(Doc, ch[:200]).save())      # loaded changes, then later ones
    later.apply_changes(ch[200:], want_patch=False)
    # a peer whose filter holds the first 200 changes: the later ones are Bloom-negative and the dependency closure runs
    peer = [sync.BloomFilter(hashes[:200])]
    return [
        ('sync_bloom_all', d, lambda: d.sync_bloom([])),
        ('sync_bloom_last_sync', d, lambda: d.sync_bloom([hashes[100]])),
        ('sync_changes_to_send', d, lambda: d.sync_changes_to_send([], peer, [])),
        ('decode_changes', d, lambda: d.decode_changes_flat(mixed)),
        ('decode_history', d, lambda: d.decode_history_flat()),
        ('encode', d, lambda: d.encode_flat(table)),
        ('history_patches', d, lambda: d.history_patches_flat([0, 1, 150, 300])),
        ('merge', local, lambda: local.merge_flat(remote)),
        ('save', later, lambda: later.save()),
    ]


def check_launches(Doc):
    got = {}
    for name, doc, call in _entry_point_calls(Doc):
        l0 = doc.launches()
        call()
        got[name] = doc.launches() - l0
    return got


def test_entry_point_launches_emu(emu_doc):
    got = check_launches(emu_doc)
    assert got == EXPECTED_LAUNCHES, got


def test_spans_zero_emu(emu_doc):
    """the emulation build has no device clock: every span reads 0"""
    for name, doc, call in _entry_point_calls(emu_doc):
        call()
        assert [getattr(doc, 'last_%s_ms' % k)() for k in SPANS] == [0.0] * len(SPANS), name


def _spans(doc):
    return {k: getattr(doc, 'last_%s_ms' % k)() for k in SPANS}


@pytest.mark.gpu
def test_device_spans_gpu(gpu_doc):
    """each call sets its own span and no other; a call that fails leaves its span at 0"""
    from automerge_classic_b200.engine import AmgError
    ch = _trace()
    d = _doc(gpu_doc, ch[:-20])
    remote = _doc(gpu_doc, ch)
    table = d.decode_changes_flat(ch[:80])
    calls = [('sync', lambda: d.sync_bloom([])), ('decode', lambda: d.decode_history_flat()), ('encode', lambda: d.encode_flat(table)),
             ('history', lambda: d.history_patches_flat([100])), ('merge', lambda: d.merge_flat(remote)), ('sync', lambda: d.sync_bloom([]))]
    for kind, call in calls:
        before = _spans(d)
        call()
        after = _spans(d)
        assert after[kind] > 0, (kind, after)
        assert {k: v for k, v in after.items() if k != kind} == {k: v for k, v in before.items() if k != kind}, (kind, before, after)
    damaged = bytearray(ch[5])
    damaged[5] ^= 0xff   # the checksum no longer matches
    failing = [('decode', lambda: d.decode_changes_flat([ch[0], bytes(damaged)])), ('encode', lambda: d.encode_flat(table.raw[:16])),
               ('history', lambda: d.history_patches_flat([len(ch) + 1]))]
    for kind, call in failing:
        before = _spans(d)
        assert before[kind] > 0
        with pytest.raises(AmgError):
            call()
        after = _spans(d)
        assert after[kind] == 0, (kind, after)
        assert {k: v for k, v in after.items() if k != kind} == {k: v for k, v in before.items() if k != kind}, (kind, before, after)
        dict(calls)[kind]()   # the next call of the kind times itself again
        assert _spans(d)[kind] > 0
