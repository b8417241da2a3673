"""The device DEFLATE decoder (inflate_tabled, csrc/inflate.cuh) on hand-built streams at its code, block and window
edges, against zlib and the oracle.

A compressor only writes the codes it likes, so the streams here come from deflate_writer.py, which writes the blocks,
code lengths and symbols each case asks for. Every stream inflates to the chunk body of a plain change: the change keeps
its magic and checksum, takes chunk type 2 and carries the stream. The body is a change header, a run of N letters 'a'
(a string value: inside the run a match at any distance back into the run copies 'a's, so lengths and distances can be
chosen freely) and the columns behind it.

Each case states the edge it is built to reach, and the test checks that claim against the writer's record of what it
wrote (block types, HLIT / HDIST / HCLEN, repeat codes, longest codes, longest match, farthest distance, the bit
position a cut falls in, the body's size against the decoder's scratch capacity). Each case states its verdict, and the
test checks it first with zlib (zlib.decompress(stream, -15): the oracle and the reference's pako inflate the same way).

Two doors: applyChanges (patch, op table, heads and getChanges([]) - the original compressed bytes - against the oracle;
on refusal the document is unchanged) and decodeChanges (the host decoder's change objects and the oracle's hash, or a
refusal). Then all accepted cases again, rebuilt for 5 000 and more authors, in one batch mixed with plain changes: on
the device the warps of k_inflate take several streams in turn and rebuild the tables another stream's block left.
The cases run on the serial emulation build by default, and with -m gpu on libamgpu.so (the only run of the table build
with 32 lanes).
"""
import zlib

import pytest

import deflate_writer as W
import parity_checks
import replay
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401

A = ord('a')
DIST1 = [1]   # one distance code of one bit: distance code 0 (distance 1) only


def _uleb(v):
    from automerge_classic_b200 import columnar
    return columnar.uleb(v)


def plain_change(i, run, msg='', all_bytes=False, key='k'):
    """a plain change of author i: a string of `run` letters 'a' under key '<key><i>' (and all 256 byte values under
    'b<i>'); returns (raw change, chunk body, offset of the run in the body)"""
    from automerge_classic_b200 import columnar
    ops = []
    if all_bytes:
        ops.append({'action': 'set', 'obj': '_root', 'key': 'b%05d' % i, 'value': bytes(range(256)), 'pred': []})
    ops.append({'action': 'set', 'obj': '_root', 'key': '%s%05d' % (key, i), 'value': 'a' * run, 'pred': []})
    # actor ids start with byte 0: the body opens with 00 10 00 (no deps, a 16-byte actor id), which back_to_start copies
    change = {'actor': '00%030x' % (i + 1), 'seq': 1, 'startOp': 1, 'time': 0, 'message': msg, 'deps': [], 'ops': ops}
    raw, _ = columnar.encode_change_raw(change, False)
    pos = 9
    while raw[pos] & 0x80:
        pos += 1
    body = raw[pos + 1:]
    return raw, body, body.rfind(b'a' * run) if run else len(body) - 2


def deflated(raw, stream):
    return raw[:8] + b'\x02' + _uleb(len(stream)) + stream


def capacity(change):
    """the scratch capacity the engine gives a stream (InflateCapKernel: 4 x the change's length + 1 024)"""
    return 4 * len(change) + 1024


# ------------------------------------------------------------------------------------------------------------ symbols
def lits(data):
    return list(data)


def run_syms(n, length=258, dist=1, first=True):
    """n letters 'a' as a literal (when `first`) and matches of `length` at `dist`; the rest as a shorter match or
    literals"""
    out, have = ([A], 1) if first and n else ([], 0)
    while n - have >= 3:
        k = min(length, n - have)
        out.append(('m', k, dist)); have += k
    return out + [A] * (n - have)


def lz(history, data):
    """greedy LZ77 of `data` behind `history` (3-byte hash, last position only, distances up to 32 768)"""
    buf = bytes(history) + bytes(data)
    last, out, i = {}, [], len(history)
    for j in range(max(0, len(history) - 32768), len(history) - 2):
        last[buf[j:j + 3]] = j
    while i < len(buf):
        k, best = buf[i:i + 3], 0
        j = last.get(k)
        if j is not None and i - j <= 32768 and len(k) == 3:
            while best < 258 and i + best < len(buf) and buf[j + best] == buf[i + best]:
                best += 1
        if best >= 3:
            out.append(('m', best, i - j))
            for t in range(i, i + best):
                last[buf[t:t + 3]] = t
            i += best
        else:
            last[k] = i
            out.append(buf[i]); i += 1
    return out


def used_lit(symbols):
    u = set()
    for s in symbols:
        u.add(s if isinstance(s, int) else W.len_code(s[1], s[3] if len(s) > 3 else None)[0])
    return sorted(u | {W.EOB})


def used_dist(symbols):
    return sorted({W.dist_code(s[2])[0] for s in symbols if not isinstance(s, int)})


def dyn_block(w, symbols, final=False, nlit=286, ndist=None, **kw):
    """a dynamic block over `symbols` with a complete code over the symbols it uses"""
    ds = used_dist(symbols)
    lit = W.complete_lengths(nlit, {}, used_lit(symbols))
    if not ds:
        dist = [0] * (ndist or 1)
    elif len(ds) == 1:
        dist = [0] * ds[0] + [1]
    else:
        dist = W.complete_lengths(max(ds) + 1 if ndist is None else ndist, {}, ds)
    w.dynamic(lit, dist, symbols, final=final, **kw)


# -------------------------------------------------------------------------------------------------------------- cases
# A case: (body spec, builder(P, N, Q) -> Writer, claims, accepted). The body spec is a dict of plain_change arguments, or
# {'size': n} for a body of exactly n bytes, or {'cap': d} for a body d bytes over the stream's scratch capacity.
# Claims: {block index: {field: value}} checked against the writer's record ('has_<field>': a subset of it, 'min_<field>':
# at least); 'stream' claims: blocks, trailing, body_len, over_cap (body length - capacity), cut (the item a cut ends in).
CASES = {}


def case(name, body, claims, accepted=True):
    def reg(fn):
        CASES[name] = (body, fn, claims, accepted)
        return fn
    return reg


def _lc(i):
    return W.LEN_BASE[i], W.LEN_BASE[i] + (1 << W.LEN_EXTRA[i]) - 1


def _dc(i):
    return W.DIST_BASE[i], W.DIST_BASE[i] + (1 << W.DIST_EXTRA[i]) - 1


# stored blocks
@case('stored_empty', {'run': 300}, {0: {'type': 'stored', 'len': 0}})
def _(P, N, Q):
    w = W.Writer(); w.stored(b''); w.fixed(lits(P) + run_syms(N) + lits(Q), final=True); return w


@case('stored_65535', {'run': 70000}, {1: {'type': 'stored', 'len': 65535}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + [A]); w.stored(b'a' * 65535)
    w.fixed(run_syms(N - 65536, first=False) + lits(Q), final=True); return w


@case('stored_in_a_row', {'run': 3000}, {'stream': {'blocks': 5}, 0: {'type': 'stored'}, 4: {'type': 'stored', 'final': True}})
def _(P, N, Q):
    body = P + b'a' * N + Q
    w, cuts = W.Writer(), [0, 40, 41, 1000, 2500, len(body)]
    for k in range(5):
        w.stored(body[cuts[k]:cuts[k + 1]], final=k == 4)
    return w


@case('stored_after_mid_byte', {'run': 500}, {0: {'type': 'fixed'}, 1: {'type': 'stored', 'mid_byte': True}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + [A, A]); w.stored(b'a' * (N - 2) + Q, final=True); return w


@case('stored_final', {'run': 500}, {1: {'type': 'stored', 'final': True, 'len': 2}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + run_syms(N)); w.stored(Q, final=True); return w


# fixed blocks
@case('fixed_all_literals', {'run': 3, 'all_bytes': True}, {0: {'type': 'fixed', 'has_lsyms': set(range(256))}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P + b'aaa' + Q), final=True); return w


LEN_EDGES = [(n, 257 + i) for i in range(28) for n in _lc(i)] + [(258, 284), (258, 285)]


@case('fixed_length_codes', {'run': 1 + sum(n for n, _ in LEN_EDGES)},
      {0: {'has_lextra': {(s, n - W.LEN_BASE[s - 257]) for n, s in LEN_EDGES}, 'longest': 258}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + [A] + [('m', n, 1, s) for n, s in LEN_EDGES] + lits(Q), final=True); return w


DIST_EDGES = [d for i in range(30) for d in _dc(i)]


@case('fixed_distance_codes', {'run': 32768 + 3 * len(DIST_EDGES)},
      {0: {'has_dextra': {(i, d - W.DIST_BASE[i]) for i in range(30) for d in _dc(i)}, 'farthest': 32768}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + run_syms(32768) + [('m', 3, d) for d in DIST_EDGES] + lits(Q), final=True); return w


@case('fixed_overlap', {'run': 2000, 'msg': 'abcdefg' * 60}, {0: {'overlap': True, 'has_dextra': {(5, 0), (0, 0)}}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lz(b'', P) + run_syms(N) + lits(Q), final=True); return w


@case('fixed_back_to_start', {'run': 300, 'msg': '\x00\x10\x00xyz'}, {0: {'back_to_start': True}})
def _(P, N, Q):
    p = P.find(P[:3], 1)
    w = W.Writer(); w.fixed(lits(P[:p]) + [('m', 3, p)] + lits(P[p + 3:]) + run_syms(N) + lits(Q), final=True); return w


# dynamic blocks
EVERY_LEN = [A] + list(range(257, 271)) + [W.EOB]   # lengths 1..14 for the first 14, 15 for the last two


@case('dynamic_every_length', {'run': 1 + sum(W.LEN_BASE[:14])},
      {1: {'type': 'dynamic', 'lit_lengths': set(range(1, 16)), 'lit_max': 15, 'has_lsyms': set(EVERY_LEN), 'hclen': 19,
           'hdist': 1, 'dist_lengths': {1}}})
def _(P, N, Q):
    lit = [0] * 271
    for k, s in enumerate(EVERY_LEN):
        lit[s] = min(k + 1, 15)
    w = W.Writer(); w.fixed(lits(P))
    w.dynamic(lit, DIST1, [A] + [('m', W.LEN_BASE[i], 1) for i in range(14)])
    w.fixed(lits(Q), final=True); return w


@case('dynamic_distance_lengths', {'run': 600 + 3 * 16},
      {1: {'dist_lengths': set(range(1, 16)), 'dist_max': 15, 'has_dsyms': set(range(16))}})
def _(P, N, Q):
    dist = [min(k + 1, 15) for k in range(16)]
    syms = run_syms(600) + [('m', 3, W.DIST_BASE[i]) for i in range(16)]
    w = W.Writer(); w.fixed(lits(P))
    w.dynamic(W.complete_lengths(286, {}, used_lit(syms)), dist, syms)
    w.fixed(lits(Q), final=True); return w


@case('dynamic_lanes_wrap', {'run': 1000},
      {0: {'min_most_one_length': 33, 'has_lit_lengths': {10, 11}, 'hdist': 1}})
def _(P, N, Q):
    syms = lits(P) + run_syms(N) + lits(Q)
    used = used_lit(syms)
    free = [s for s in range(286) if s not in used]
    lit = W.complete_lengths(286, {**{s: 10 for s in free[:70]}, **{s: 11 for s in free[70:140]}}, used)
    w = W.Writer(); w.dynamic(lit, DIST1, syms, final=True); return w


@case('dynamic_all_286', {'run': 1000}, {0: {'lit_used': 286, 'hlit': 286}})
def _(P, N, Q):
    syms = lits(P) + run_syms(N) + lits(Q)
    lit = W.complete_lengths(286, {}, used_lit(syms) + list(range(286)))
    w = W.Writer(); w.dynamic(lit, DIST1, syms, final=True); return w


@case('dynamic_hlit_257', {'run': 40}, {0: {'hlit': 257, 'longest': 0}})
def _(P, N, Q):
    syms = lits(P + b'a' * N + Q)
    w = W.Writer(); w.dynamic(W.complete_lengths(257, {}, used_lit(syms)), DIST1, syms, final=True); return w


@case('dynamic_one_distance_code', {'run': 3000}, {0: {'hdist': 1, 'dist_used': 1, 'dist_max': 1, 'code_left': (0, 1 << 14)}})
def _(P, N, Q):
    syms = lits(P) + run_syms(N) + lits(Q)
    w = W.Writer(); w.dynamic(W.complete_lengths(286, {}, used_lit(syms)), DIST1, syms, final=True); return w


@case('dynamic_no_distance_code', {'run': 40}, {0: {'hdist': 1, 'dist_used': 0, 'longest': 0}})
def _(P, N, Q):
    syms = lits(P + b'a' * N + Q)
    w = W.Writer(); w.dynamic(W.complete_lengths(286, {}, used_lit(syms)), [0], syms, final=True); return w


@case('dynamic_hclen_19', {'run': 3000}, {0: {'hclen': 19}})
def _(P, N, Q):
    syms = lits(P) + run_syms(N) + lits(Q)
    lit = W.complete_lengths(286, {}, used_lit(syms))
    assert max(lit) < 15
    w = W.Writer(); w.dynamic(lit, DIST1, syms, final=True, hclen=19); return w


REPEAT_FIXED = {**{s: 9 for s in range(3, 10)}, **{s: 9 for s in range(21, 25)}, 35: 9}


@case('dynamic_repeats', {'run': 5 + 3 * 300},
      {1: {'has_repeats': {(16, 3), (16, 6), (17, 3), (17, 10), (18, 11), (18, 138)}, 'cross': True, 'hdist': 5,
           'dist_used': 1}})
def _(P, N, Q):
    syms = [A] * 5 + [('m', 3, 5)] * 300
    lit = W.complete_lengths(286, REPEAT_FIXED, [A, W.EOB, 257], spare=[40, 41, 42, 43, 44, 45])
    w = W.Writer(); w.fixed(lits(P)); w.dynamic(lit, [0, 0, 0, 0, 1], syms); w.fixed(lits(Q), final=True); return w


@case('dynamic_eob_only_1bit', {'run': 300}, {0: {'type': 'dynamic', 'lit_used': 1, 'lit_max': 1, 'hlit': 257}})
def _(P, N, Q):
    w = W.Writer(); w.dynamic([0] * 256 + [1], [0], [])
    w.fixed(lits(P) + run_syms(N) + lits(Q), final=True); return w


# streams
@case('hundred_blocks', {'run': 3000}, {'stream': {'blocks': 100}, 50: {'type': 'dynamic'}, 99: {'final': True}})
def _(P, N, Q):
    body = P + b'a' * N + Q
    w, step = W.Writer(), -(-len(body) // 100)
    for k in range(100):
        piece, final = body[k * step:(k + 1) * step], k == 99
        syms = lz(body[:k * step], piece)
        (w.stored(piece, final) if k % 3 == 0 else w.fixed(syms, final) if k % 3 == 1 else dyn_block(w, syms, final))
    return w


@case('matches_into_earlier_blocks', {'run': 3000}, {1: {'into_earlier': True}, 2: {'into_earlier': True, 'type': 'dynamic'}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + run_syms(1000))
    w.fixed([('m', 100, 900)] + run_syms(900, first=False))
    dyn_block(w, [('m', 258, 2000)] + run_syms(N - 2258, first=False) + lits(Q), final=True); return w


@case('bytes_after_final', {'run': 300}, {'stream': {'trailing': 7}})
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + run_syms(N) + lits(Q), final=True); w.trail(b'\x00\xff\x13junk'); return w


# sizes: the scratch capacity (the over-capacity body is decoded a second time, into place) and the LEB128 width of the
# length the inflated change is given
def _sized(P, N, Q):
    w = W.Writer(); w.stored(P); w.fixed(run_syms(N)); w.stored(Q, final=True); return w


case('cap_exact', {'cap': 0}, {'stream': {'over_cap': 0}})(_sized)
case('cap_plus_one', {'cap': 1}, {'stream': {'over_cap': 1}})(_sized)
for _n in (127, 128, 16383, 16384):
    case('body_%d' % _n, {'size': _n}, {'stream': {'body_len': _n}})(_sized)


# ------------------------------------------------------------------------------------------------------- refused cases
def _lit_block(P, N, Q, **kw):
    syms = lits(P + b'a' * N + Q)
    return syms, W.complete_lengths(286, {}, used_lit(syms))


@case('oversubscribed', {'run': 40}, {0: {'code_left': ('<', 0)}}, accepted=False)
def _(P, N, Q):
    syms, lit = _lit_block(P, N, Q)
    lit[next(s for s in range(286) if lit[s] == 0)] = 1   # (no symbols: their codes would not fit)
    w = W.Writer(); w.dynamic(lit, DIST1, [], final=True, eob=False); return w


@case('one_distance_code_of_2', {'run': 40}, {0: {'dist_used': 1, 'dist_max': 2, 'longest': 0}}, accepted=False)
def _(P, N, Q):
    syms, lit = _lit_block(P, N, Q)
    w = W.Writer(); w.dynamic(lit, [2], syms, final=True); return w


@case('eob_only_of_2', {'run': 300}, {0: {'lit_used': 1, 'lit_max': 2}}, accepted=False)
def _(P, N, Q):
    w = W.Writer(); w.dynamic([0] * 256 + [2], [0], [])
    w.fixed(lits(P) + run_syms(N) + lits(Q), final=True); return w


@case('no_eob', {'run': 40}, {0: {'eob_code': False}}, accepted=False)
def _(P, N, Q):
    syms = lits(P + b'a' * N + Q)
    lit = W.complete_lengths(286, {}, sorted(set(syms)), spare=range(257, 286))
    w = W.Writer(); w.dynamic(lit, DIST1, syms, final=True, eob=False); return w


@case('repeat_16_first', {'run': 40}, {0: {'seq_first': (16, 3)}}, accepted=False)
def _(P, N, Q):
    syms, lit = _lit_block(P, N, Q)
    seq = W.rle(lit + DIST1)
    w = W.Writer(); w.dynamic(lit, DIST1, syms, final=True, seq=[(16, 3)] + seq); return w


@case('repeat_past_end', {'run': 40}, {0: {'min_seq_total': 288}}, accepted=False)
def _(P, N, Q):
    syms, lit = _lit_block(P, N, Q)
    seq = W.rle(lit) + [(17, 3)]   # HLIT + 1 lengths: the run of three goes two past the end
    w = W.Writer(); w.dynamic(lit, DIST1, syms, final=True, seq=seq); return w


for _hl, _hd in ((287, 1), (288, 1), (257, 31), (257, 32)):
    def _mk(hl, hd):
        def build(P, N, Q):
            syms = lits(P + b'a' * N + Q)
            lit = W.complete_lengths(hl, {}, used_lit(syms))
            w = W.Writer(); w.dynamic(lit, [0] * (hd - 1) + [1], syms, final=True); return w
        return build
    case('hlit_%d_hdist_%d' % (_hl, _hd), {'run': 40}, {0: {'hlit': _hl, 'hdist': _hd}}, accepted=False)(_mk(_hl, _hd))


@case('hclen_4', {'run': 40}, {0: {'hclen': 4, 'eob_code': False}}, accepted=False)
def _(P, N, Q):
    # with code-length codes 16, 17, 18 and 0 alone every length is 0: there is no end-of-block code
    w = W.Writer(); w.dynamic([0] * 257, [0], [], final=True, eob=False); w.fixed(lits(P + b'a' * N + Q), final=True); return w


for _s in (286, 287):
    case('fixed_symbol_%d' % _s, {'run': 40}, {0: {'has_lsyms': {_s}}}, accepted=False)(
        lambda P, N, Q, s=_s: _w(lambda w: w.fixed(lits(P) + [('L', s)], final=True)))
for _s in (30, 31):
    case('fixed_distance_%d' % _s, {'run': 40}, {0: {'has_dsyms': {_s}}}, accepted=False)(
        lambda P, N, Q, s=_s: _w(lambda w: w.fixed(lits(P) + [('L', 257), ('D', s)], final=True)))


def _w(fn):
    w = W.Writer(); fn(w); return w


@case('distance_too_far', {'run': 40}, {0: {'too_far': True}}, accepted=False)
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + [('m', 3, len(P) + 1)], final=True); return w


@case('block_type_3', {'run': 40}, {0: {'type': 'raw'}}, accepted=False)
def _(P, N, Q):
    w = W.Writer(); w.block_type(3); w.bits(0, 13); return w


@case('stored_nlen_mismatch', {'run': 40}, {0: {'type': 'stored'}}, accepted=False)
def _(P, N, Q):
    body = P + b'a' * N + Q
    w = W.Writer(); w.stored(body, final=True, nlen=len(body) ^ 0xfffe); return w


@case('no_final_block', {'run': 300}, {'stream': {'blocks': 1}, 0: {'final': False}}, accepted=False)
def _(P, N, Q):
    w = W.Writer(); w.fixed(lits(P) + run_syms(N) + lits(Q)); return w


def _cut_base(P, N, Q):
    """a dynamic block with long codes and far distances, then a stored block"""
    syms = lits(P) + run_syms(25000) + [('m', 3, W.DIST_BASE[i] + 1) for i in range(30)]
    lit = W.complete_lengths(286, {}, used_lit(syms))
    w = W.Writer(); w.dynamic(lit, W.complete_lengths(30, {}, list(range(30))), syms); w.stored(b'a' * (N - 25090) + Q, final=True)
    return w


for _what in ('header', 'lengths', 'code', 'extra', 'payload'):
    case('cut_in_' + _what, {'run': 25090 + 3000}, {'stream': {'cut': _what}}, accepted=False)(
        lambda P, N, Q, what=_what: (_cut_base(P, N, Q), what))


def _spans(rec, what):
    if what in ('header', 'lengths', 'payload'):
        return [rec[what]] if what in rec else []
    return rec[what + '_spans']


def cut_at(w, what):
    """the byte count at which the stream ends inside an item of kind `what` (some but not all of its bits)"""
    for rec in w.blocks:
        for s, e in _spans(rec, what):
            k = s // 8 + 1
            if s < 8 * k < e:
                return k
    raise AssertionError('no %s straddles a byte boundary' % what)


# ------------------------------------------------------------------------------------------------------------- building
_ARGS = {}


def _exact(size):
    """(run, message) of a body of exactly `size` bytes"""
    for run in range(max(3, size - 80), size + 1):
        for m in range(8):
            if len(plain_change(0, run, 'm' * m)[1]) == size:
                return run, 'm' * m
    raise AssertionError(size)


def _args(name):
    """plain_change arguments (run, message, all_bytes) of a case: the same body length for every author"""
    if name not in _ARGS:
        spec, build = CASES[name][:2]
        if 'size' in spec:
            _ARGS[name] = _exact(spec['size']) + (False,)
        elif 'cap' in spec:
            target = 2000
            for _ in range(20):
                run, msg = _exact(target)
                raw, body, r = plain_change(0, run, msg)
                want = capacity(deflated(raw, build(body[:r], run, body[r + run:]).getvalue())) + spec['cap']
                if want == target:
                    break
                target = want
            else:
                raise AssertionError('no body of the capacity found')
            _ARGS[name] = (run, msg, False)
        else:
            _ARGS[name] = (spec['run'], spec.get('msg', ''), spec.get('all_bytes', False))
    return _ARGS[name]


def build_case(name, i=0):
    """(deflated change, plain change, writer, claims context) of case `name` for author i"""
    build, accepted = CASES[name][1], CASES[name][3]
    n, msg, all_bytes = _args(name)
    raw, body, r = plain_change(i, n, msg, all_bytes)
    got = build(body[:r], n, body[r + n:])
    w, what = got if isinstance(got, tuple) else (got, None)
    stream = w.getvalue()
    if what is not None:
        stream = stream[:cut_at(w, what)]
    if accepted:
        assert bytes(w.out) == body, (name, 'the writer does not produce the body')
    change = deflated(raw, stream)
    ctx = {'blocks': len(w.blocks), 'trailing': w.trailing, 'body_len': len(body), 'over_cap': len(body) - capacity(change),
           'cut': what}
    return change, raw, w, ctx, stream


def check_claims(name, w, ctx):
    claims = CASES[name][2]
    for where, cl in claims.items():
        rec = ctx if where == 'stream' else w.blocks[where]
        for key, want in cl.items():
            if key.startswith('has_'):
                assert want <= rec[key[4:]], (name, where, key, want - rec[key[4:]])
            elif key.startswith('min_'):
                assert rec[key[4:]] >= want, (name, where, key, rec[key[4:]], want)
            elif key == 'code_left' and want[0] == '<':
                assert rec['code_left'][0] < want[1], (name, where, rec['code_left'])
            else:
                assert rec[key] == want, (name, where, key, rec[key], want)


def zlib_verdict(stream):
    try:
        return zlib.decompress(stream, -15)
    except zlib.error:
        return None


# ---------------------------------------------------------------------------------------------------------------- doors
BASE_ACTOR = 'ff' * 16


def _base():
    from automerge_classic_b200 import columnar
    return columnar.encode_change_raw({'actor': BASE_ACTOR, 'seq': 1, 'startOp': 1, 'time': 0, 'message': '', 'deps': [],
                                       'ops': [{'action': 'set', 'obj': '_root', 'key': 'base', 'value': 1, 'pred': []}]},
                                      False)[0]


def _snapshot(g):
    return sorted(g.heads()), g.clock(), g.max_op(), replay.decode(g.get_patch()), g.save()


def door_apply(Doc, oracle_mod, change, accepted):
    from automerge_classic_b200.engine import AmgError
    o, g = oracle_mod.OracleDoc(), Doc()
    o.apply_changes([_base()]); g.apply_changes([_base()])
    before = _snapshot(g)
    try:
        po = o.apply_changes([change])
    except oracle_mod.OracleError:
        po = None
    assert (po is not None) == accepted, 'the oracle disagrees with zlib'
    try:
        pg = g.apply_changes([change])
    except AmgError:
        pg = None
    if not accepted:
        assert pg is None, 'the engine accepts a stream zlib refuses'
        assert _snapshot(g) == before
        return
    assert pg is not None, 'the engine refuses a stream zlib accepts'
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    parity_checks._dump_equal(g, o)
    assert sorted(g.heads()) == sorted(o.heads())
    assert g.get_changes([]) == o.get_changes([])
    assert change in g.get_changes([])


def door_decode(Doc, oracle_mod, change, accepted):
    from automerge_classic_b200 import columnar
    from automerge_classic_b200.engine import AmgError
    try:
        exp = oracle_mod.decode_change(change)
    except oracle_mod.OracleError:
        exp = None
    assert (exp is not None) == accepted, 'the oracle disagrees with zlib'
    try:
        got = Doc().decode_changes_flat([change]).to_changes()
    except AmgError:
        got = None
    if not accepted:
        assert got is None, 'the engine decodes a stream zlib refuses'
        return
    assert got is not None, 'the engine refuses a stream zlib accepts'
    assert got == [columnar.decode_change(change)]
    assert got[0]['hash'] == exp['hash']


def run_case(Doc, oracle_mod, name):
    change, raw, w, ctx, stream = build_case(name)
    check_claims(name, w, ctx)
    accepted = CASES[name][3]
    body = zlib_verdict(stream)
    assert (body is not None) == accepted, ('zlib', name)
    if accepted:
        assert parity_checks._inflated(change) == raw
    door_apply(Doc, oracle_mod, change, accepted)
    door_decode(Doc, oracle_mod, change, accepted)


BATCH = 5000


def run_batch(Doc, oracle_mod):
    """every accepted case, rebuilt for new authors until there are BATCH DEFLATEd changes, one plain change after every
    third, in one applyChanges call"""
    from automerge_classic_b200 import columnar
    names = [n for n, c in CASES.items() if c[3]]
    batch, i = [], 0
    while i < BATCH:
        for name in names:
            change, raw, w, ctx, stream = build_case(name, i)
            assert zlib_verdict(stream) is not None
            batch.append(change)
            if i % 3 == 0:
                batch.append(columnar.encode_change_raw(
                    {'actor': '11%030x' % i, 'seq': 1, 'startOp': 1, 'time': 0, 'message': '', 'deps': [],
                     'ops': [{'action': 'set', 'obj': '_root', 'key': 'p%05d' % i, 'value': 'x' * (i % 50), 'pred': []}]},
                    False)[0])
            i += 1
    assert sum(c[8] == 2 for c in batch) >= BATCH
    o, g = oracle_mod.OracleDoc(), Doc()
    po, pg = o.apply_changes(batch), g.apply_changes(batch)
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    parity_checks._dump_equal(g, o)
    assert sorted(g.heads()) == sorted(o.heads())
    assert g.get_changes([]) == o.get_changes([])
    assert sorted(g.get_changes([])) == sorted(batch)
    got = g.decode_changes_flat(batch).to_changes()
    assert got == [columnar.decode_change(c) for c in batch]


@pytest.mark.parametrize('name', list(CASES))
def test_stream_emu(emu_doc, oracle_mod, name):
    run_case(emu_doc, oracle_mod, name)


def test_batch_emu(emu_doc, oracle_mod):
    run_batch(emu_doc, oracle_mod)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_stream_gpu(gpu_doc, oracle_mod, name):
    run_case(gpu_doc, oracle_mod, name)


@pytest.mark.gpu
def test_batch_gpu(gpu_doc, oracle_mod):
    run_batch(gpu_doc, oracle_mod)
