"""A raw DEFLATE (RFC 1951) writer for tests: it writes exactly the blocks, codes and symbols the caller asks for, including
ones a compressor never writes (single-symbol codes, 15-bit codes, repeats across the literal/distance boundary, codes a
decoder must refuse). Next to the bytes it keeps a record of what each block holds, and the bytes a decoder must produce.

Symbols of a Huffman block: an int 0-255 is a literal; ('m', length, distance) a match, with ('m', 258, distance, 284) for
the length 258 written as code 284 with extra bits 31; ('L', sym) and ('D', sym) a bare literal/length or distance code
(refused streams). The end-of-block code follows unless the block is written with eob=False."""

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [max(0, i // 2 - 1) for i in range(30)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32   # codes 30 and 31 exist in the fixed code but never occur in a valid stream (RFC 1951 3.2.6)
EOB = 256


def len_code(length, sym=None):
    """(symbol, extra bit count, extra value) of a match length"""
    if sym is None:
        sym = 285 if length == 258 else 257 + max(i for i in range(28) if LEN_BASE[i] <= length)
    i = sym - 257
    extra = length - LEN_BASE[i]
    assert 0 <= extra < (1 << LEN_EXTRA[i]) or (i == 28 and extra == 0), (length, sym)
    return sym, LEN_EXTRA[i], extra


def dist_code(d):
    i = max(i for i in range(30) if DIST_BASE[i] <= d)
    assert d - DIST_BASE[i] < (1 << DIST_EXTRA[i]), d
    return i, DIST_EXTRA[i], d - DIST_BASE[i]


def canonical(lengths):
    """the canonical code of every symbol (RFC 1951 3.2.2), None for unused ones"""
    mx = max(lengths) if lengths else 0
    count = [0] * (mx + 2)
    for ln in lengths:
        if ln:
            count[ln] += 1
    nxt, code = [0] * (mx + 2), 0
    for b in range(1, mx + 1):
        code = (code + count[b - 1]) << 1 if b > 1 else 0
        nxt[b] = code
    out = []
    for ln in lengths:
        if ln:
            out.append((nxt[ln], ln)); nxt[ln] += 1
        else:
            out.append(None)
    return out


def kraft_left(lengths, maxlen=15):
    """2^maxlen minus the code space the lengths take: 0 = complete, > 0 incomplete, < 0 over-subscribed"""
    return (1 << maxlen) - sum(1 << (maxlen - ln) for ln in lengths if ln)


def complete_lengths(n, fixed, fill, maxlen=15, spare=None):
    """code lengths for an alphabet of n symbols: `fixed` maps symbols to lengths, the symbols of `fill` (in order) take the
    rest of the code space so that the code is complete, shortest codes first. Where `fill` has too few symbols for the
    space left, unused symbols are added: from `spare`, else from the top of the alphabet."""
    lens = [0] * n
    for s, ln in fixed.items():
        lens[s] = ln
    left = kraft_left(lens, maxlen)
    assert left >= 0, 'over-subscribed'
    pieces = [1 << b for b in range(maxlen, -1, -1) if left >> b & 1]
    fill = list(dict.fromkeys(s for s in fill if s not in fixed))
    spare = [s for s in (range(n - 1, -1, -1) if spare is None else spare) if s not in fixed and s not in fill]
    while len(pieces) > len(fill):
        fill.append(spare.pop(0))
    while len(pieces) < len(fill):
        pieces.sort(reverse=True)
        assert pieces[0] > 1, 'too many symbols for the code space'
        p = pieces.pop(0)
        pieces += [p // 2, p // 2]
    pieces.sort(reverse=True)
    for s, p in zip(fill, pieces):
        lens[s] = maxlen - (p.bit_length() - 1)
    assert kraft_left(lens, maxlen) == 0
    return lens


def rle(lengths):
    """code-length sequence with repeats where they apply: 18 / 17 for runs of zeros, 16 after a length for its repeats"""
    seq, i, n = [], 0, len(lengths)
    while i < n:
        v, j = lengths[i], i
        while j < n and lengths[j] == v:
            j += 1
        run = j - i
        if v == 0:
            while run >= 11:
                k = min(run, 138); seq.append((18, k)); run -= k
            if run >= 3:
                seq.append((17, run)); run = 0
            seq += [0] * run
        else:
            seq.append(v); run -= 1
            while run >= 3:
                k = min(run, 6); seq.append((16, k)); run -= k
            seq += [v] * run
        i = j
    return seq


def expand(seq):
    out = []
    for s in seq:
        if isinstance(s, int):
            out.append(s)
        elif s[0] == 16:
            out += out[-1:] * s[1]
        else:
            out += [0] * s[1]
    return out


class BitWriter:
    def __init__(self):
        self.buf, self.acc, self.n = bytearray(), 0, 0

    @property
    def pos(self):
        return 8 * len(self.buf) + self.n

    def bits(self, v, n):
        assert 0 <= v < (1 << n) or (n == 0 and v == 0), (v, n)
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.buf.append(self.acc & 0xff); self.acc >>= 8; self.n -= 8

    def code(self, c):
        code, ln = c
        self.bits(int(format(code, '0%db' % ln)[::-1], 2), ln)   # Huffman codes go most significant bit first

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def getvalue(self):
        return bytes(self.buf) + (bytes([self.acc]) if self.n else b'')


class Writer:
    def __init__(self):
        self.w = BitWriter()
        self.blocks = []
        self.out = bytearray()   # what a decoder produces
        self.trailing = 0

    def _begin(self, kind, final, btype):
        rec = {'type': kind, 'final': bool(final), 'start_bit': self.w.pos, 'mid_byte': self.w.pos % 8 != 0,
               'out_start': len(self.out)}
        self.blocks.append(rec)
        self.w.bits(int(final), 1)
        self.w.bits(btype, 2)
        return rec

    def stored(self, data, final=False, nlen=None):
        rec = self._begin('stored', final, 0)
        self.w.align()
        n = len(data)
        self.w.bits(n, 16)
        self.w.bits(n ^ 0xffff if nlen is None else nlen, 16)
        rec['payload'] = (self.w.pos, self.w.pos + 8 * n)
        self.w.buf += data   # (byte-aligned here)
        self.out += data
        rec['len'] = n
        rec['end_bit'] = self.w.pos

    def block_type(self, btype, final=True):
        """a block header alone (type 3 is reserved)"""
        self._begin('raw', final, btype)

    def fixed(self, symbols, final=False, eob=True):
        rec = self._begin('fixed', final, 1)
        self._symbols(rec, FIXED_LIT, FIXED_DIST, symbols, eob)

    def dynamic(self, lit, dist, symbols, final=False, seq=None, cl=None, hclen=None, hlit=None, hdist=None, eob=True):
        """lit / dist: the code lengths; seq: the code-length sequence (default rle(lit + dist)); cl: the code-length code's
        lengths by symbol (default: a complete code over the symbols seq uses); hclen: code-length code lengths written"""
        rec = self._begin('dynamic', final, 2)
        hlit = len(lit) if hlit is None else hlit
        hdist = len(dist) if hdist is None else hdist
        seq = rle(list(lit) + list(dist)) if seq is None else seq
        used = sorted({s if isinstance(s, int) else s[0] for s in seq})
        if cl is None:
            cl = complete_lengths(19, {}, used if len(used) > 1 else used + [0 if used != [0] else 1], maxlen=7)
        if hclen is None:
            hclen = 19
            while hclen > 4 and cl[CL_ORDER[hclen - 1]] == 0:
                hclen -= 1
        self.w.bits(hlit - 257, 5)
        self.w.bits(hdist - 1, 5)
        self.w.bits(hclen - 4, 4)
        for i in range(hclen):
            self.w.bits(cl[CL_ORDER[i]], 3)
        rec.update(hlit=hlit, hdist=hdist, hclen=hclen, header=(rec['start_bit'], self.w.pos))
        clc = canonical(cl)
        start, idx, repeats, cross = self.w.pos, 0, set(), False
        for s in seq:
            sym, k = (s, 1) if isinstance(s, int) else s
            self.w.code(clc[sym])
            if sym >= 16:
                self.w.bits(k - (11 if sym == 18 else 3), {16: 2, 17: 3, 18: 7}[sym])
                repeats.add((sym, k))
                cross = cross or idx < hlit < idx + k
            idx += k
        rec.update(lengths=(start, self.w.pos), repeats=repeats, cross=cross, cl=list(cl), seq_first=seq[0] if seq else None,
                   seq_total=idx, eob_code=len(lit) > EOB and lit[EOB] > 0)
        if expand(seq) == list(lit) + list(dist):
            rec['code_left'] = (kraft_left(lit), kraft_left(dist))
        self._symbols(rec, lit, dist, symbols, eob)

    def _symbols(self, rec, lit, dist, symbols, eob):
        lc, dc = canonical(list(lit)), canonical(list(dist))
        ll = [x for x in lit if x]
        dl = [x for x in dist if x]
        rec.update(lit_max=max(ll, default=0), dist_max=max(dl, default=0), lit_lengths=set(ll), dist_lengths=set(dl),
                   lit_used=len(ll), dist_used=len(dl), most_one_length=max((ll.count(v) for v in set(ll)), default=0),
                   longest=0, farthest=0, overlap=False, back_to_start=False, lsyms=set(), dsyms=set(), lextra=set(),
                   dextra=set(), code_spans=[], extra_spans=[], into_earlier=False, too_far=False)
        out, w = self.out, self.w

        def put_code(c):
            s = w.pos; w.code(c); rec['code_spans'].append((s, w.pos))

        def put_extra(v, n):
            if n:
                s = w.pos; w.bits(v, n); rec['extra_spans'].append((s, w.pos))

        rec['symbols_start'] = w.pos
        for s in list(symbols) + ([('L', EOB)] if eob else []):
            if isinstance(s, int):
                put_code(lc[s]); out.append(s); rec['lsyms'].add(s)
            elif s[0] == 'L':
                put_code(lc[s[1]]); rec['lsyms'].add(s[1])
            elif s[0] == 'D':
                put_code(dc[s[1]]); rec['dsyms'].add(s[1])
            else:
                length, d = s[1], s[2]
                sym, nb, ev = len_code(length, s[3] if len(s) > 3 else None)
                ds, dnb, dv = dist_code(d)
                put_code(lc[sym]); put_extra(ev, nb); put_code(dc[ds]); put_extra(dv, dnb)
                rec['lsyms'].add(sym); rec['dsyms'].add(ds); rec['lextra'].add((sym, ev)); rec['dextra'].add((ds, dv))
                rec['longest'] = max(rec['longest'], length); rec['farthest'] = max(rec['farthest'], d)
                rec['overlap'] = rec['overlap'] or d < length
                rec['back_to_start'] = rec['back_to_start'] or d == len(out)
                rec['into_earlier'] = rec['into_earlier'] or d > len(out) - rec['out_start']
                rec['too_far'] = rec['too_far'] or d > len(out)
                if d <= len(out):
                    for _ in range(length):
                        out.append(out[-d])
        rec['end_bit'] = w.pos

    def bits(self, v, n):
        self.w.bits(v, n)

    def trail(self, data):
        """bytes after the final block"""
        self.w.align()
        for b in data:
            self.w.bits(b, 8)
        self.trailing += len(data)

    def getvalue(self):
        return self.w.getvalue()
