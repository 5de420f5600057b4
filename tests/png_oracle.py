"""Numpy restatement of the PNG encoder of next3d_b200/csrc/png.cu (DESIGN.md section 3.6): the same decisions, the same bytes.

A file is the signature, IHDR (8-bit RGB, no interlace), one IDAT chunk holding a zlib stream, and IEND.  The zlib stream:
  * rows filtered with the filter (0-4) of least sum of |int8(filtered byte)|, ties to the lower filter number;
  * the filtered bytes cut into stripes of `stripe_rows(W)` rows; each stripe is one deflate block of its own bit stream: dynamic
    Huffman codes over a greedy LZ77 parse, or stored blocks when those are no larger.  Every stripe but the last ends with an
    empty stored block (a sync flush), so stripes concatenate on byte boundaries; matches may reach into earlier stripes;
  * the LZ77 candidates are fixed distances (`candidates`), taken longest first and in list order on ties, so that every
    position's matches are known without the parse;
  * Huffman code lengths from a two-queue Huffman construction over (frequency, symbol)-sorted leaves, with frequencies halved
    until the longest code fits the limit (15 bits; 7 for the code-length code);
  * the Adler-32 of the filtered bytes and, per chunk, a CRC-32 computed over 4096-byte segments and combined with x^(8n) mod P.
"""
import struct

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'
STRIPE_BYTES = 32768         # target filtered bytes per stripe
MAX_DIST = 32768
MAX_MATCH = 258
STORED_MAX = 65535
CRC_SEGMENT = 4096

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in range(2)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]

# symbol and extra-bit count of every match length 3..258 and distance 1..32768
LEN_SYM = np.zeros(MAX_MATCH + 1, np.int64)
for _k, _b in enumerate(LEN_BASE):
    LEN_SYM[_b:] = _k
LEN_SYM[MAX_MATCH] = 28
DIST_SYM = np.zeros(MAX_DIST + 1, np.int64)
for _k, _b in enumerate(DIST_BASE):
    DIST_SYM[_b:] = _k


def row_bytes(width):
    return 3 * width + 1


def stripe_rows(width):
    """Rows per stripe: a function of the row length alone."""
    return max(1, STRIPE_BYTES // row_bytes(width))


def candidates(width):
    """LZ77 candidate distances in priority order: the previous byte, pixel and second pixel, the byte above and the pixels
    above-left and above-right.  Distances beyond the 32 KiB window are dropped."""
    bpr = row_bytes(width)
    return [d for d in (1, 3, 6, bpr, bpr - 3, bpr + 3) if 1 <= d <= MAX_DIST]


def stored_bytes(n):
    """Stored-block size of n raw bytes: 5 header bytes per block of at most 65535."""
    return n + 5 * -(-n // STORED_MAX)


def capacity(height, width):
    """Largest file the encoder can write for the size: a stored stripe is never exceeded."""
    bpr, rows = row_bytes(width), stripe_rows(width)
    full, last = divmod(height, rows)
    body = full * stored_bytes(rows * bpr) + (stored_bytes(last * bpr) if last else 0)
    return len(SIGNATURE) + 25 + 12 + 2 + body + 4 + 12


# ---------------------------------------------------------------------------------------------------------------- filters
def filter_rows(img):
    """[H, W, 3] uint8 -> ([H] filter types, [H, 3W + 1] uint8 filtered rows with the filter byte first)."""
    H, W, _ = img.shape
    x = img.reshape(H, 3 * W).astype(np.int16)
    up = np.vstack([np.zeros((1, 3 * W), np.int16), x[:-1]])
    left = np.hstack([np.zeros((H, 3), np.int16), x[:, :-3]])
    ul = np.hstack([np.zeros((H, 3), np.int16), up[:, :-3]])
    p = left + up - ul
    pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
    paeth = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
    cand = np.stack([x, x - left, x - up, x - ((left + up) >> 1), x - paeth]) & 0xff         # [5, H, 3W]
    cost = np.minimum(cand, 256 - cand).sum(axis=2)                                          # sum of |int8|
    ftype = np.argmin(cost, axis=0)                                                          # first minimum: lower filter
    rows = cand[ftype, np.arange(H)].astype(np.uint8)
    return ftype, np.hstack([ftype.astype(np.uint8)[:, None], rows])


# ---------------------------------------------------------------------------------------------------------------- LZ77
def match_lengths(buf, s0, s1, dists):
    """[len(dists), s1 - s0] match length at every position of the stripe for every candidate (0 where out of the window)."""
    n = s1 - s0
    out = np.zeros((len(dists), n), np.int64)
    pos = np.arange(s0, s1)
    for k, d in enumerate(dists):
        lo = max(s0, d)                                   # first position whose candidate lies inside the image
        if lo >= s1:
            continue
        eq = buf[lo:s1] == buf[lo - d:s1 - d]
        # index of the first mismatch at or after each position (s1 if none)
        idx = np.where(~eq, np.arange(lo, s1), s1)
        nxt = np.minimum.accumulate(idx[::-1])[::-1]
        out[k, lo - s0:] = np.minimum(nxt - pos[lo - s0:], MAX_MATCH)
    return out


def parse(buf, s0, s1, dists):
    """Greedy parse of buf[s0:s1]: at each position the longest candidate match (first candidate on ties) if it is at least 3
    bytes, else a literal.  -> (value, distance) int64 arrays of the tokens in order: (byte, 0) for a literal, (length,
    distance) for a match."""
    n = s1 - s0
    L = match_lengths(buf, s0, s1, dists)
    best = L.argmax(axis=0)
    blen = L[best, np.arange(n)]
    ok = np.flatnonzero(blen >= 3)
    starts, p = [], 0
    while True:                                      # one step per match; the literals between matches are skipped over
        j = np.searchsorted(ok, p)
        if j == len(ok):
            break
        q = int(ok[j])
        starts.append(q)
        p = q + int(blen[q])
    starts = np.array(starts, np.int64)
    covered = np.zeros(n + 1, np.int64)
    np.add.at(covered, starts, 1)
    np.add.at(covered, starts + blen[starts], -1)
    lit = np.flatnonzero(np.cumsum(covered[:n]) == 0)
    pos = np.sort(np.concatenate([lit, starts]))
    is_match = np.zeros(n, bool)
    is_match[starts] = True
    m = is_match[pos]
    dist_of = np.asarray(dists, np.int64)[best[pos]]
    value = np.where(m, blen[pos], buf[s0 + pos].astype(np.int64))
    return value, np.where(m, dist_of, 0)


# ---------------------------------------------------------------------------------------------------------------- Huffman
def huffman_lengths(freq):
    """Code lengths of a Huffman code for the nonzero frequencies: leaves sorted by (frequency, symbol), the two lightest of the
    leaf queue and the node queue merged (a leaf first on equal weight), depths read from the root."""
    syms = sorted((f, s) for s, f in enumerate(freq) if f)
    n = len(syms)
    lengths = [0] * len(freq)
    w = [f for f, _ in syms]                 # node weights: leaves 0..n-1, then internal nodes n..2n-2
    parent = [0] * (2 * n - 1)
    i, j = 0, n                              # heads of the leaf queue and the internal-node queue
    for k in range(n, 2 * n - 1):
        kids = []
        for _ in range(2):
            if i < n and (j >= k or w[i] <= w[j]):
                kids.append(i)
                i += 1
            else:
                kids.append(j)
                j += 1
        w.append(w[kids[0]] + w[kids[1]])
        parent[kids[0]] = parent[kids[1]] = k
    depth = [0] * (2 * n - 1)
    for k in range(2 * n - 3, -1, -1):
        depth[k] = depth[parent[k]] + 1
    for k, (_, s) in enumerate(syms):
        lengths[s] = depth[k]
    return lengths


def limited_lengths(freq, limit):
    """Huffman code lengths of at most `limit` bits.  At least two symbols get codes (symbols 0 and 1 are given a count of 1
    while fewer than two are used); while the longest code is too long, every nonzero frequency f becomes (f + 1) // 2."""
    f = [int(v) for v in freq]
    for s in (0, 1):
        if sum(1 for v in f if v) < 2:
            f[s] = max(f[s], 1)
    while True:
        lengths = huffman_lengths(f)
        if max(lengths) <= limit:
            return lengths
        f = [(v + 1) >> 1 for v in f]


def canonical_codes(lengths):
    """Deflate's canonical codes, bit-reversed for least-significant-bit-first output."""
    bl = [0] * 16
    for ln in lengths:
        bl[ln] += 1
    bl[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    codes = [0] * len(lengths)
    for s, ln in enumerate(lengths):
        if ln:
            c = nxt[ln]
            nxt[ln] += 1
            codes[s] = int(format(c, f'0{ln}b')[::-1], 2)
    return codes


def rle_lengths(seq):
    """Code-length symbols (symbol, extra value) for a sequence of code lengths: runs of zeros as 18 (11-138) then 17 (3-10),
    other runs as the length then 16 (3-6 repeats) while at least 3 remain; what is left is written as it is."""
    out, i, n = [], 0, len(seq)
    while i < n:
        v, r = seq[i], 1
        while i + r < n and seq[i + r] == v:
            r += 1
        i += r
        if v == 0:
            while r >= 11:
                k = min(r, 138)
                out.append((18, k - 11))
                r -= k
            if r >= 3:
                out.append((17, r - 3))
                r = 0
            out.extend([(0, 0)] * r)
        else:
            out.append((v, 0))
            r -= 1
            while r >= 3:
                k = min(r, 6)
                out.append((16, k - 3))
                r -= k
            out.extend([(v, 0)] * r)
    return out


CL_EXTRA = {16: 2, 17: 3, 18: 7}


class BitWriter:
    def __init__(self):
        self.vals, self.nbits = [], []

    def put(self, v, n):
        if n:
            self.vals.append(int(v))
            self.nbits.append(int(n))

    def put_array(self, vals, nbits):
        keep = nbits > 0
        self.vals.extend(vals[keep].tolist())
        self.nbits.extend(nbits[keep].tolist())

    @property
    def bits(self):
        return int(sum(self.nbits))

    def tobytes(self):
        """The bits least significant first, zero-padded to a byte."""
        n = np.asarray(self.nbits, np.int64)
        v = np.asarray(self.vals, np.uint64)
        if len(n) == 0:
            return b''
        owner = np.repeat(np.arange(len(n)), n)
        k = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
        bit = ((v[owner] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return np.packbits(bit, bitorder='little').tobytes()


def dynamic_block(lit, dist, final):
    """One dynamic-Huffman block (BFINAL = final) of the tokens (parse's arrays) plus end of block -> BitWriter."""
    lf, df = [0] * 286, [0] * 30
    m = dist > 0
    lsym = np.where(m, 257 + LEN_SYM[np.where(m, lit, 3)], lit)
    dsym = DIST_SYM[dist[m]]
    for s, c in zip(*np.unique(lsym, return_counts=True)):
        lf[s] = int(c)
    for s, c in zip(*np.unique(dsym, return_counts=True)):
        df[s] = int(c)
    lf[256] = 1
    ll, dl = limited_lengths(lf, 15), limited_lengths(df, 15)
    hlit = max(257, max(s for s in range(286) if ll[s]) + 1)
    hdist = max(1, max(s for s in range(30) if dl[s]) + 1)
    cls = rle_lengths(ll[:hlit] + dl[:hdist])
    cf = [0] * 19
    for s, _ in cls:
        cf[s] += 1
    cl = limited_lengths(cf, 7)
    hclen = max(4, max(k for k in range(19) if cl[CL_ORDER[k]]) + 1)
    lc, dc, cc = canonical_codes(ll), canonical_codes(dl), canonical_codes(cl)

    w = BitWriter()
    w.put(int(final) | (2 << 1), 3)
    w.put(hlit - 257, 5)
    w.put(hdist - 1, 5)
    w.put(hclen - 4, 4)
    for k in range(hclen):
        w.put(cl[CL_ORDER[k]], 3)
    for s, e in cls:
        w.put(cc[s], cl[s])
        if s in CL_EXTRA:
            w.put(e, CL_EXTRA[s])
    # tokens: one value of at most 48 bits each (code, length extra, distance code, distance extra)
    lc_a, ll_a, dc_a, dl_a = (np.array(a, np.int64) for a in (lc, ll, dc, dl))
    lb = np.array(LEN_BASE, np.int64)[np.clip(lsym - 257, 0, 28)]
    le = np.array(LEN_EXTRA, np.int64)[np.clip(lsym - 257, 0, 28)]
    ds = DIST_SYM[dist]
    db, de = np.array(DIST_BASE, np.int64)[ds], np.array(DIST_EXTRA, np.int64)[ds]
    val, nb = lc_a[lsym], ll_a[lsym]
    val = val | np.where(m, (lit - lb) << nb, 0)
    nb = nb + np.where(m, le, 0)
    val = val | np.where(m, dc_a[ds] << nb, 0)
    nb = nb + np.where(m, dl_a[ds], 0)
    val = val | np.where(m, (dist - db) << nb, 0)
    nb = nb + np.where(m, de, 0)
    w.put_array(val, nb)
    w.put(lc[256], ll[256])
    return w


def stored_blocks(data, final):
    out, n = bytearray(), len(data)
    for o in range(0, n, STORED_MAX):
        k = min(STORED_MAX, n - o)
        out.append(int(final and o + k == n))
        out += struct.pack('<HH', k, k ^ 0xffff)
        out += data[o:o + k]
    return bytes(out)


def encode_stripe(buf, s0, s1, dists, last):
    """-> (bytes of the stripe, True if stored)."""
    w = dynamic_block(*parse(buf, s0, s1, dists), last)
    dyn = (w.bits + 7) // 8 if last else (w.bits + 3 + 7) // 8 + 4
    if dyn > stored_bytes(s1 - s0):
        return stored_blocks(buf[s0:s1].tobytes(), last), True
    if not last:
        w.put(0, 3)                                  # empty stored block: BFINAL 0, BTYPE 00, then padding and LEN / NLEN
    out = w.tobytes()
    if not last:
        out += b'\x00\x00\xff\xff'
    assert len(out) == dyn
    return out, False


# ---------------------------------------------------------------------------------------------------------------- checksums
def adler32(data):
    x = np.frombuffer(data, np.uint8).astype(np.int64)
    n = len(x)
    a = (1 + int(x.sum())) % 65521
    b = (n + int(((n - np.arange(n)) % 65521 * x % 65521).sum())) % 65521
    return (b << 16) | a


_CRC_TABLE = np.zeros(256, np.uint32)
for _i in range(256):
    _c = _i
    for _ in range(8):
        _c = (_c >> 1) ^ (0xEDB88320 if _c & 1 else 0)
    _CRC_TABLE[_i] = _c


def multmodp(a, b):
    """a(x) * b(x) mod P(x) on reflected 32-bit polynomials (bit 31 is x^0)."""
    m, p = 1 << 31, 0
    while True:
        if a & m:
            p ^= b
            if a & (m - 1) == 0:
                return p
        m >>= 1
        b = (b >> 1) ^ 0xEDB88320 if b & 1 else b >> 1


def x8nmodp(n):
    """x^(8n) mod P(x), reflected."""
    r, sq = 1 << 31, 1 << 23                           # x^0; x^8 (x^(8 * 2^k) by repeated squaring)
    while n:
        if n & 1:
            r = multmodp(sq, r)
        sq = multmodp(sq, sq)
        n >>= 1
    return r


def crc32(data):
    """CRC-32 of the bytes: unconditioned CRCs of 4096-byte segments (all segments advanced one byte at a time together), then
    combined in order as crc = crc * x^(8 * len(segment)) + crc(segment)."""
    x = np.frombuffer(data, np.uint8)
    n = len(x)
    nseg = max(1, -(-n // CRC_SEGMENT))
    pad = np.zeros(nseg * CRC_SEGMENT, np.uint8)
    pad[:n] = x
    seg = pad.reshape(nseg, CRC_SEGMENT)
    lens = np.minimum(CRC_SEGMENT, n - CRC_SEGMENT * np.arange(nseg))
    c = np.zeros(nseg, np.uint32)
    for k in range(CRC_SEGMENT):
        live = lens > k
        nc = _CRC_TABLE[(c ^ seg[:, k]) & 0xff] ^ (c >> np.uint32(8))
        c = np.where(live, nc, c)
    crc = 0xffffffff                                   # the initial register, shifted through the whole message below
    for k in range(nseg):
        crc = multmodp(x8nmodp(int(lens[k])), crc) ^ int(c[k])
    return crc ^ 0xffffffff


def chunk(kind, payload):
    return struct.pack('>I', len(payload)) + kind + payload + struct.pack('>I', crc32(kind + payload))


# ---------------------------------------------------------------------------------------------------------------- files
def zlib_stream(img, info=None):
    H, W, _ = img.shape
    _, rows = filter_rows(img)
    buf = rows.reshape(-1)
    bpr, sr = row_bytes(W), stripe_rows(W)
    dists = candidates(W)
    out = bytearray(b'\x78\x01')
    stored = []
    for r0 in range(0, H, sr):
        r1 = min(H, r0 + sr)
        data, st = encode_stripe(buf, r0 * bpr, r1 * bpr, dists, r1 == H)
        out += data
        stored.append(st)
    out += struct.pack('>I', adler32(buf.tobytes()))
    if info is not None:
        info['stored'] = stored
    return bytes(out)


def encode(img, info=None):
    """[H, W, 3] uint8 -> PNG file bytes.  info (a dict, optional) receives 'stored': per stripe, whether it was stored."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    assert img.ndim == 3 and img.shape[2] == 3 and img.shape[0] > 0 and img.shape[1] > 0
    H, W, _ = img.shape
    ihdr = struct.pack('>IIBBBBB', W, H, 8, 2, 0, 0, 0)
    return SIGNATURE + chunk(b'IHDR', ihdr) + chunk(b'IDAT', zlib_stream(img, info)) + chunk(b'IEND', b'')
