"""FLAC (RFC 9639) restated in numpy for the tests: an encoder that can emit every coding tool on demand, with a libFLAC-like
default, and a plain decoder.  Neither is used by the product; the GPU decoder (csrc/flac.cu) is checked against them and against
the PCM that was encoded.

The encoder writes each frame as a list of (value, width) fields and packs all frames of a file in one vectorised pass (a field
of up to 64 significant bits and any width; a Rice code is the one field (1 << k | low, q + 1 + k)).  The CRC-16 of every frame is
computed together by combining per-byte CRCs pairwise (CRC(A B) = CRC(A) x^(8|B|) + CRC(B) mod P; leading zero bytes leave a CRC
of initial value 0 unchanged, so frames are left-padded to a common power-of-two length).
"""
from __future__ import annotations

import numpy as np

BLOCK_CODES = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13, 16384: 14, 32768: 15}
RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
DEPTH_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}
ASSIGN = {'independent': None, 'left_side': 8, 'side_right': 9, 'mid_side': 10}
PADDING, APPLICATION, SEEKTABLE, VORBIS_COMMENT, CUESHEET, PICTURE = 1, 2, 3, 4, 5, 6


def _crc8_table():
    t = np.zeros(256, np.uint16)
    for i in range(256):
        c = i
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
        t[i] = c
    return t


def _crc16_table():
    t = np.zeros(256, np.uint32)
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        t[i] = c
    return t


CRC8, CRC16 = _crc8_table(), _crc16_table()


def crc8(data: bytes) -> int:
    c = 0
    for b in data:
        c = int(CRC8[c ^ b])
    return c


def crc16(data: bytes) -> int:
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ int(CRC16[(c >> 8) ^ b])
    return c


def _mulmod(a: int, b: int) -> int:
    """a b mod x^16 + x^15 + x^2 + 1 (carry-less)."""
    r = 0
    for i in range(16):
        if b >> i & 1:
            r ^= a << i
    for i in range(31, 15, -1):
        if r >> i & 1:
            r ^= 0x18005 << (i - 16)
    return r


def crc16_batch(frames) -> list:
    """CRC-16 (polynomial 0x8005, initial 0) of every byte string of a list, vectorised across the strings."""
    if not frames:
        return []
    L = 1 << max(1, int(np.ceil(np.log2(max(len(f) for f in frames) or 1))))
    buf = np.zeros((len(frames), L), np.uint8)
    for i, f in enumerate(frames):
        if len(f):
            buf[i, L - len(f):] = np.frombuffer(f, np.uint8)
    v = CRC16[buf]
    level = 0                                   # each entry of v covers 2^level bytes
    while v.shape[1] > 1:
        hi, lo = _shift_tables(level)
        left = v[:, 0::2]
        v = hi[left >> 8] ^ lo[left & 0xFF] ^ v[:, 1::2]
        level += 1
    return [int(c) for c in v[:, 0]]


_SHIFT = []


def _shift_tables(level):
    """Tables of (c x^(8 2^level)) mod P for the high and the low byte of c."""
    while len(_SHIFT) <= level:
        x = 1
        for _ in range(8 << len(_SHIFT)):
            x = _mulmod(x, 2)
        _SHIFT.append((np.array([_mulmod(i << 8, x) for i in range(256)], np.uint32),
                       np.array([_mulmod(i, x) for i in range(256)], np.uint32)))
    return _SHIFT[level]


# ---------------------------------------------------------------------------------------------------------------- bit writing
def pack_fields(vals, widths) -> np.ndarray:
    """MSB-first bits of fields (value, width) -> uint8 bits (0/1).  Only the low 64 bits of a value are significant; the bits of a
    wider field above them are zeros (a unary run)."""
    vals = np.asarray(vals, dtype=np.uint64)
    widths = np.asarray(widths, dtype=np.int64)
    ends = np.cumsum(widths)
    bits = np.zeros(int(ends[-1]) if len(ends) else 0, np.uint8)
    if not len(bits):
        return bits
    top = int(vals.max()).bit_length()
    for j in range(min(top, 64)):
        sel = widths > j
        bits[ends[sel] - 1 - j] = ((vals[sel] >> np.uint64(j)) & np.uint64(1)).astype(np.uint8)
    return bits


class Fields:
    def __init__(self):
        self.v, self.w = [], []

    def put(self, value, width):
        self.v.append(np.asarray([int(value) & ((1 << 64) - 1)], np.uint64))
        self.w.append(np.asarray([width], np.int64))

    def put_signed(self, value, width):
        self.put(int(value) & ((1 << width) - 1) if width else 0, width)

    def put_array(self, values, width):
        a = np.asarray(values, np.int64)
        self.v.append((a & np.int64((1 << width) - 1)).astype(np.uint64) if width < 64 else a.astype(np.uint64))
        self.w.append(np.full(len(a), width, np.int64))

    def put_codes(self, vals, widths):
        self.v.append(np.asarray(vals, np.uint64))
        self.w.append(np.asarray(widths, np.int64))

    def bits(self) -> int:
        return int(sum(w.sum() for w in self.w))

    def arrays(self):
        if not self.v:
            return np.zeros(0, np.uint64), np.zeros(0, np.int64)
        return np.concatenate(self.v), np.concatenate(self.w)


# ---------------------------------------------------------------------------------------------------------------- prediction
def fixed_residual(x, order):
    x = np.asarray(x, np.int64)
    r = x.copy()
    for _ in range(order):
        r = np.diff(r)
    return r  # len(x) - order values: the residual after the warm-up


def lpc_coefficients(x, order):
    """Least-squares-like LPC by autocorrelation of a Welch-windowed copy and Levinson-Durbin -> float64 a (x[n] ~ sum a_j x[n-1-j])."""
    x = np.asarray(x, np.float64)
    n = len(x)
    w = 1.0 - ((np.arange(n) - (n - 1) / 2.0) / ((n + 1) / 2.0)) ** 2
    y = x * w
    r = np.array([np.dot(y[:n - k], y[k:]) for k in range(order + 1)])
    if r[0] == 0:
        return np.zeros(order)
    r[0] *= 1.0 + 1e-9
    a = np.zeros(order)
    err = r[0]
    for i in range(order):
        k = (r[i + 1] - np.dot(a[:i], r[i:0:-1])) / err
        a[:i] = a[:i] - k * a[:i][::-1]
        a[i] = k
        err *= 1.0 - k * k
        if err <= 0:
            break
    return a


def quantize_lpc(a, precision, shift=None):
    """-> (int coefficients within `precision` signed bits, shift 0..15)."""
    lim = 1 << (precision - 1)
    if shift is None:
        m = np.max(np.abs(a)) if len(a) else 0.0
        shift = precision - 1 - (int(np.floor(np.log2(m))) + 1 if m > 0 else 0)
        shift = int(min(max(shift, 0), 15))
    q = np.clip(np.round(np.asarray(a) * (1 << shift)), -lim, lim - 1).astype(np.int64)
    return q, shift


def lpc_residual(x, q, shift):
    x = np.asarray(x, np.int64)
    order = len(q)
    n = len(x)
    pred = np.zeros(n - order, np.int64)
    for j in range(order):
        pred += int(q[j]) * x[order - 1 - j:n - 1 - j]
    return x[order:] - (pred >> shift)


# ---------------------------------------------------------------------------------------------------------------- residual coding
def _zigzag(r):
    r = np.asarray(r, np.int64)
    return ((r << 1) ^ (r >> 63)).astype(np.uint64)


def residual_fields(f: Fields, r, block, order, method=None, porder=None, escape=False, max_porder=6):
    """Partitioned Rice coding of the residual r (block - order values).  method 0 Rice / 1 Rice2 (None: Rice2 when a parameter
    above 14 pays), porder None: the cheapest order <= max_porder the block allows, escape: every partition escaped.  The bit
    counts of every parameter and partition come from sums over the finest partitions."""
    r = np.asarray(r, np.int64)
    u = _zigzag(r)
    orders = [porder] if porder is not None else [p for p in range(max_porder + 1) if block % (1 << p) == 0 and (block >> p) >= order]
    meths = [method] if method is not None else [0, 1]
    pmax = max(orders)
    psize = block >> pmax
    bounds = np.array([0] + [psize * i - order for i in range(1, (1 << pmax) + 1)])
    counts = np.diff(bounds)
    K = 31
    if escape:
        mags = np.array([int(np.abs(r[a:b]).max(initial=0)).bit_length() for a, b in zip(bounds[:-1], bounds[1:])])
    else:
        sums = np.zeros((K, 1 << pmax), np.int64)
        nz = counts > 0
        for k in range(K):
            sums[k, nz] = np.add.reduceat((u >> np.uint64(k)).astype(np.int64), bounds[:-1][nz])
    best = None
    for p in orders:
        g = 1 << (pmax - p)
        cnt = counts.reshape(1 << p, g).sum(1)
        for m in meths:
            if escape:
                w = mags.reshape(1 << p, g).max(1)
                w = np.where(w > 0, w + 1, 0)
                params = [('esc', int(v)) for v in w]
                cost = int(((5 if m else 4) + 5 + w * cnt).sum())
            else:
                kmax = 30 if m else 14
                c = sums[:kmax + 1].reshape(kmax + 1, 1 << p, g).sum(2) + cnt[None, :] * (np.arange(kmax + 1)[:, None] + 1)
                ks = c.argmin(0)
                params = [('rice', int(k)) for k in ks]
                cost = int(c.min(0).sum()) + (5 if m else 4) * (1 << p)
            if best is None or cost < best[0]:
                best = (cost, params, p, m)
    _, params, p, m = best
    bounds = [0] + [(block >> p) * i - order for i in range(1, (1 << p) + 1)]
    f.put(m, 2)
    f.put(p, 4)
    for i, (kind, k) in enumerate(params):
        seg_r, seg_u = r[bounds[i]:bounds[i + 1]], u[bounds[i]:bounds[i + 1]]
        if kind == 'esc':
            f.put(31 if m else 15, 5 if m else 4)
            f.put(k, 5)
            if k:
                f.put_array(seg_r, k)
        else:
            f.put(k, 5 if m else 4)
            q = (seg_u >> np.uint64(k)).astype(np.int64)
            low = seg_u & np.uint64((1 << k) - 1)
            f.put_codes((np.uint64(1) << np.uint64(k)) | low, q + 1 + k)


# ---------------------------------------------------------------------------------------------------------------- subframes
def subframe_fields(f: Fields, x, bits, spec):
    """One subframe of the int samples x at `bits` bits.  spec: dict(type='constant'|'verbatim'|'fixed'|'lpc'|'auto', order,
    precision, shift, wasted (None: all the common trailing zero bits; forced values must divide every sample), method, porder,
    escape, max_porder)."""
    x = np.asarray(x, np.int64)
    block = len(x)
    kind = spec.get('type', 'auto')
    wasted = spec.get('wasted')
    if wasted is None:
        nz = x[x != 0]
        wasted = 0 if not len(nz) else min(int((nz & -nz).min()).bit_length() - 1, bits - 1)
    assert 0 <= wasted < bits and not np.any(x & ((1 << wasted) - 1)), 'forced wasted bits must divide every sample'
    x = x >> wasted
    b = bits - wasted
    if kind == 'auto':
        kind = 'constant' if np.all(x == x[0]) else 'lpc'
    f.put(0, 1)
    if kind == 'constant':
        assert np.all(x == x[0])
        f.put(0, 6)
    elif kind == 'verbatim':
        f.put(1, 6)
    elif kind == 'fixed':
        f.put(8 + spec['order'], 6)
    else:
        order = min(spec.get('order', 8), block)
        f.put(31 + order, 6)
    if wasted:
        f.put(1, 1)
        f.put(1, wasted)                               # wasted - 1 zeros, then a one
    else:
        f.put(0, 1)
    res = dict(method=spec.get('method'), porder=spec.get('porder'), escape=spec.get('escape', False),
               max_porder=spec.get('max_porder', 6))
    if kind == 'constant':
        f.put_signed(x[0], b)
    elif kind == 'verbatim':
        f.put_array(x, b)
    elif kind == 'fixed':
        order = spec['order']
        f.put_array(x[:order], b)
        residual_fields(f, fixed_residual(x, order), block, order, **res)
    else:
        prec = spec.get('precision', 12)
        q, shift = quantize_lpc(lpc_coefficients(x, order), prec, spec.get('shift'))
        f.put_array(x[:order], b)
        f.put(prec - 1, 4)
        f.put_signed(shift, 5)
        f.put_array(q, prec)
        residual_fields(f, lpc_residual(x, q, shift), block, order, **res)


def _coded_number(n: int) -> bytes:
    if n < 0x80:
        return bytes([n])
    for nbytes, lead, cap in ((2, 0xC0, 11), (3, 0xE0, 16), (4, 0xF0, 21), (5, 0xF8, 26), (6, 0xFC, 31), (7, 0xFE, 36)):
        if n < 1 << cap:
            out = [0x80 | (n >> (6 * i) & 0x3F) for i in range(nbytes - 1)][::-1]
            return bytes([lead | (n >> (6 * (nbytes - 1)))] + out)
    raise ValueError(n)


def frame_header(block, rate, channels_code, bps, number, variable, bs_form='table', rate_form='table', bps_form='table') -> bytes:
    """A frame header with its CRC-8.  bs_form 'table' | '8' | '16'; rate_form 'table' | 'streaminfo' | 'khz' | 'hz' | 'tens';
    bps_form 'table' | 'streaminfo'."""
    tail = b''
    if bs_form == 'table' and block in BLOCK_CODES:
        bc = BLOCK_CODES[block]
    elif bs_form in ('table', '8') and block <= 256:
        bc, tail = 6, bytes([block - 1])
    else:
        bc, tail = 7, (block - 1).to_bytes(2, 'big')
    if rate_form == 'streaminfo':
        rc = 0
    elif rate_form == 'khz':
        rc, tail = 12, tail + bytes([rate // 1000])
    elif rate_form == 'hz':
        rc, tail = 13, tail + rate.to_bytes(2, 'big')
    elif rate_form == 'tens':
        rc, tail = 14, tail + (rate // 10).to_bytes(2, 'big')
    elif rate in RATE_CODES:
        rc = RATE_CODES[rate]
    else:
        rc = 0
    dc = DEPTH_CODES.get(bps, 0) if bps_form == 'table' else 0
    h = bytes([0xFF, 0xF8 | int(variable), bc << 4 | rc, channels_code << 4 | dc << 1]) + _coded_number(number) + tail
    return h + bytes([crc8(h)])


def _stereo_cost(ch):
    return int(np.abs(fixed_residual(ch, 2)).sum()) if len(ch) > 2 else 0


def encode(pcm, rate, bps, block_size=4096, variable=False, spec=None, stereo='auto', header=None, blocks=None,
           metadata='default', streaminfo_total=True, frame_spec=None) -> bytes:
    """int PCM (N, C) (or (N,)) at `bps` bits -> a FLAC file.

    block_size: an int (the last frame takes the rest), or a list of frame sizes (summing to N) for variable blocking or a
    non-uniform fixed stream.  variable: variable blocking (sample numbers).  spec: subframe spec for every subframe (see
    subframe_fields); frame_spec(frame, channel) -> spec overrides it.  stereo: 'auto' (the cheapest of the four assignments per
    frame, libFLAC's choice by an order-2 estimate), 'independent', 'left_side', 'side_right', 'mid_side'.  header: dict of
    frame_header forms.  metadata: 'default' (VORBIS_COMMENT, SEEKTABLE, PADDING), None, or a list of (type, payload bytes).
    streaminfo_total False writes an unknown (0) total."""
    x = np.asarray(pcm, np.int64)
    if x.ndim == 1:
        x = x[:, None]
    n, C = x.shape
    assert 1 <= C <= 8 and 4 <= bps <= 32
    lo, hi = -(1 << (bps - 1)), (1 << (bps - 1)) - 1
    assert x.min(initial=0) >= lo and x.max(initial=0) <= hi
    sizes = list(blocks) if blocks is not None else [min(block_size, n - s) for s in range(0, n, block_size)]
    assert sum(sizes) == n and all(s >= 1 for s in sizes)
    spec = dict(spec or {})
    header = dict(header or {})
    frames, start = [], 0
    vals, widths, frame_bits = [], [], []
    for fi, bs in enumerate(sizes):
        seg = x[start:start + bs]
        mode = stereo if C == 2 else 'independent'
        if mode == 'auto':
            l, r = seg[:, 0], seg[:, 1]
            side = l - r
            mid = (l + r) >> 1
            costs = {'independent': _stereo_cost(l) + _stereo_cost(r), 'left_side': _stereo_cost(l) + _stereo_cost(side),
                     'side_right': _stereo_cost(side) + _stereo_cost(r), 'mid_side': _stereo_cost(mid) + _stereo_cost(side)}
            mode = min(costs, key=costs.get)
        code = ASSIGN[mode]
        if code is None:
            chans, bits = [seg[:, c] for c in range(C)], [bps] * C
            code = C - 1
        else:
            l, r = seg[:, 0], seg[:, 1]
            side = l - r
            chans = {8: [l, side], 9: [side, r], 10: [(l + r) >> 1, side]}[code]
            bits = {8: [bps, bps + 1], 9: [bps + 1, bps], 10: [bps, bps + 1]}[code]
        number = start if variable else fi
        h = frame_header(bs, rate, code, bps, number, variable, header.get('bs_form', 'table'), header.get('rate_form', 'table'),
                         header.get('bps_form', 'table'))
        f = Fields()
        f.put_array(np.frombuffer(h, np.uint8).astype(np.int64), 8)
        for c in range(C):
            subframe_fields(f, chans[c], bits[c], frame_spec(fi, c) if frame_spec else spec)
        pad = (-f.bits()) % 8
        if pad:
            f.put(0, pad)
        v, w = f.arrays()
        vals.append(v)
        widths.append(w)
        frame_bits.append(int(w.sum()))
        start += bs
    packed = np.packbits(pack_fields(np.concatenate(vals), np.concatenate(widths))).tobytes()
    ends = np.cumsum(frame_bits) // 8
    bodies = [packed[a:b] for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]
    crcs = crc16_batch(bodies)
    frames = b''.join(b + c.to_bytes(2, 'big') for b, c in zip(bodies, crcs))
    non_last = sizes[:-1] or sizes
    min_b = min(non_last) if variable or blocks is not None else sizes[0]
    max_b = max(sizes)
    info = streaminfo(max(16, min(min_b, max_b)) if len(sizes) > 1 else max(16, sizes[0]), max(16, max_b), rate, C, bps,
                      n if streaminfo_total else 0)
    return flac_file(info, default_metadata(n) if metadata == 'default' else (metadata or [])) + frames


def streaminfo(min_block, max_block, rate, channels, bps, total) -> bytes:
    v = (min_block << 16 | max_block) << 48                   # min / max frame size 0: unknown
    head = v.to_bytes(10, 'big')
    packed = (rate << 44) | ((channels - 1) << 41) | ((bps - 1) << 36) | total
    return head + packed.to_bytes(8, 'big') + bytes(16)


def default_metadata(n_samples):
    vendor = b'flac_oracle'
    comment = len(vendor).to_bytes(4, 'little') + vendor + (1).to_bytes(4, 'little') + b'\x0b\x00\x00\x00TITLE=tests'
    seek = b''.join(p.to_bytes(8, 'big') + (0).to_bytes(8, 'big') + (0).to_bytes(2, 'big') for p in (0,)) + \
        b'\xff' * 8 + bytes(10)                               # one point and one placeholder
    return [(VORBIS_COMMENT, comment), (SEEKTABLE, seek), (PADDING, bytes(8192))]


def flac_file(info: bytes, blocks) -> bytes:
    out = [b'fLaC']
    allb = [(0, info)] + list(blocks)
    for i, (t, payload) in enumerate(allb):
        last = 0x80 if i == len(allb) - 1 else 0
        out.append(bytes([last | t]) + len(payload).to_bytes(3, 'big') + payload)
    return b''.join(out)


# ---------------------------------------------------------------------------------------------------------------- plain decoder
class _Bits:
    def __init__(self, data: bytes, pos: int = 0):
        self.d, self.p = data, pos * 8

    def read(self, n):
        if n == 0:
            return 0
        a, b = self.p >> 3, (self.p + n + 7) >> 3
        if b > len(self.d):
            raise ValueError('truncated')
        v = int.from_bytes(self.d[a:b], 'big')
        v = (v >> ((b << 3) - self.p - n)) & ((1 << n) - 1)
        self.p += n
        return v

    def signed(self, n):
        v = self.read(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self):
        z = 0
        while self.read(1) == 0:
            z += 1
        return z


def _subframe(br: _Bits, block, bits):
    if br.read(1):
        raise ValueError('subframe padding bit')
    t = br.read(6)
    wasted = br.unary() + 1 if br.read(1) else 0
    b = bits - wasted
    if t == 0:
        out = [br.signed(b)] * block
    elif t == 1:
        out = [br.signed(b) for _ in range(block)]
    else:
        if 8 <= t <= 12:
            order, lpc = t - 8, False
        elif t >= 32:
            order, lpc = t - 31, True
        else:
            raise ValueError(f'reserved subframe type {t}')
        out = [br.signed(b) for _ in range(order)]
        if lpc:
            prec = br.read(4)
            if prec == 15:
                raise ValueError('invalid LPC precision')
            shift = br.signed(5)
            if shift < 0:
                raise ValueError('negative LPC shift')
            coef = [br.signed(prec + 1) for _ in range(order)]
        method, porder = br.read(2), br.read(4)
        if method > 1:
            raise ValueError('reserved residual coding')
        pb, esc = (5, 31) if method else (4, 15)
        res = []
        for p in range(1 << porder):
            cnt = (block >> porder) - (order if p == 0 else 0)
            k = br.read(pb)
            if k == esc:
                w = br.read(5)
                res += [br.signed(w) if w else 0 for _ in range(cnt)]
            else:
                for _ in range(cnt):
                    u = (br.unary() << k) | br.read(k)
                    res.append((u >> 1) ^ -(u & 1))
        for i, r in enumerate(res):
            t_ = order + i
            if lpc:
                pred = sum(coef[j] * out[t_ - 1 - j] for j in range(order)) >> shift
            else:
                o = out
                pred = (0, o[t_ - 1] if order else 0, 2 * o[t_ - 1] - o[t_ - 2] if order > 1 else 0,
                        3 * o[t_ - 1] - 3 * o[t_ - 2] + o[t_ - 3] if order > 2 else 0,
                        4 * o[t_ - 1] - 6 * o[t_ - 2] + 4 * o[t_ - 3] - o[t_ - 4] if order > 3 else 0)[order]
            out.append(r + pred)
    return [v << wasted for v in out]


def parse_streaminfo(data: bytes):
    if data[:4] != b'fLaC':
        raise ValueError('no fLaC magic')
    pos, info = 4, None
    while True:
        t, last, ln = data[pos] & 0x7F, data[pos] >> 7, int.from_bytes(data[pos + 1:pos + 4], 'big')
        body = data[pos + 4:pos + 4 + ln]
        if t == 0:
            v = int.from_bytes(body[10:18], 'big')
            info = dict(min_block=int.from_bytes(body[0:2], 'big'), max_block=int.from_bytes(body[2:4], 'big'), rate=v >> 44,
                        channels=(v >> 41 & 7) + 1, bps=(v >> 36 & 31) + 1, total=v & ((1 << 36) - 1))
        pos += 4 + ln
        if last:
            return info, pos


def decode(data: bytes):
    """A FLAC file -> (int64 PCM (total, channels), STREAMINFO dict).  Checks the CRC-8, CRC-16 and frame numbers."""
    info, pos = parse_streaminfo(data)
    chans = [[] for _ in range(info['channels'])]
    done, fi = 0, 0
    while done < info['total']:
        h0 = pos
        if data[pos] != 0xFF or data[pos + 1] & 0xFE != 0xF8:
            raise ValueError(f'lost sync at frame {fi}')
        variable = data[pos + 1] & 1
        bc, rc = data[pos + 2] >> 4, data[pos + 2] & 15
        cc, dc = data[pos + 3] >> 4, data[pos + 3] >> 1 & 7
        p = pos + 4
        lead = data[p]
        nb = 1 if lead < 0x80 else {0xC0: 2, 0xE0: 3, 0xF0: 4, 0xF8: 5, 0xFC: 6, 0xFE: 7}[
            max(k for k in (0xC0, 0xE0, 0xF0, 0xF8, 0xFC, 0xFE) if lead >= k)]
        num = lead if nb == 1 else lead & (0x7F >> nb)
        for i in range(1, nb):
            num = num << 6 | data[p + i] & 0x3F
        p += nb
        if bc == 1:
            block = 192
        elif bc <= 5:
            block = 576 << (bc - 2)
        elif bc == 6:
            block, p = data[p] + 1, p + 1
        elif bc == 7:
            block, p = int.from_bytes(data[p:p + 2], 'big') + 1, p + 2
        else:
            block = 256 << (bc - 8)
        p += {12: 1, 13: 2, 14: 2}.get(rc, 0)
        if crc8(data[h0:p]) != data[p]:
            raise ValueError(f'CRC-8 at frame {fi}')
        if num != (done if variable else fi):
            raise ValueError(f'frame number at frame {fi}')
        bps = {0: info['bps'], 1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}[dc]
        br = _Bits(data, p + 1)
        n_ch = cc + 1 if cc < 8 else 2
        sub = [_subframe(br, block, bps + (1 if (cc, c) in ((8, 1), (9, 0), (10, 1)) else 0)) for c in range(n_ch)]
        if cc == 8:
            sub[1] = [a - b for a, b in zip(sub[0], sub[1])]
        elif cc == 9:
            sub[0] = [a + b for a, b in zip(sub[0], sub[1])]
        elif cc == 10:
            m = [(a << 1) | (b & 1) for a, b in zip(sub[0], sub[1])]
            sub = [[(a + b) >> 1 for a, b in zip(m, sub[1])], [(a - b) >> 1 for a, b in zip(m, sub[1])]]
        br.p = (br.p + 7) & ~7
        end = (br.p >> 3) + 2
        if crc16(data[h0:end - 2]) != int.from_bytes(data[end - 2:end], 'big'):
            raise ValueError(f'CRC-16 at frame {fi}')
        for c in range(n_ch):
            chans[c] += sub[c]
        pos, done, fi = end, done + block, fi + 1
    return np.array(chans, np.int64).T.reshape(info['total'], info['channels']), info


# ---------------------------------------------------------------------------------------------------------------- test signals
def speech_like(n, channels, bps, rate, seed, silence=True):
    """Seeded speech-like int PCM (n, channels): a few harmonics of a gliding F0 plus noise, with stretches of digital silence,
    channels correlated (as a stereo recording is), at about -6 dBFS."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    f0 = 110 + 60 * np.sin(2 * np.pi * 0.7 * t + rng.uniform(0, 6))
    ph = 2 * np.pi * np.cumsum(f0) / rate
    base = sum(rng.uniform(0.2, 1.0) / h * np.sin(h * ph + rng.uniform(0, 6)) for h in range(1, 8))
    env = 0.5 + 0.5 * np.sin(2 * np.pi * 2.5 * t + rng.uniform(0, 6)) ** 2
    out = np.empty((n, channels))
    for c in range(channels):
        out[:, c] = base * env * rng.uniform(0.6, 1.0) + rng.standard_normal(n) * 0.01 + 0.05 * np.roll(base, 7 * c + 1)
    out /= max(np.abs(out).max(), 1e-9) * 2
    full = (1 << (bps - 1)) - 1
    pcm = np.round(out * full).astype(np.int64)
    if silence and n > 64:
        a = int(rng.integers(0, n // 3))
        pcm[a:a + n // 8] = 0
    return np.clip(pcm, -full - 1, full)


def write_wav(path, pcm, rate, bps):
    """The int PCM as a WAV file read_wav reads back to x 2^-(bps - 1): 8-bit unsigned for bps <= 8, 16-bit for <= 16, else
    24-bit left-justified in 32-bit, each left-justified."""
    import scipy.io.wavfile
    x = np.asarray(pcm, np.int64)
    if bps <= 8:
        data = ((x << (8 - bps)) + 128).astype(np.uint8)
    elif bps <= 16:
        data = (x << (16 - bps)).astype('<i2')
    else:
        data = (x << (32 - bps)).astype('<i4')
    scipy.io.wavfile.write(str(path), rate, data[:, 0] if data.ndim == 2 and data.shape[1] == 1 else data)


# ---------------------------------------------------------------------------------------------------------------- tool matrix
def tool_matrix():
    """[(case id, int PCM (N, C), rate, bps, encode kwargs)]: every coding tool and header code form the decoder supports, on
    seeded speech-like PCM with digital silence."""
    cases = []

    def add(name, n, C, bps, rate=22050, seed=None, pcm=None, **kw):
        x = speech_like(n, C, bps, rate, seed if seed is not None else len(cases)) if pcm is None else pcm
        cases.append((name, x, rate, bps, kw))

    for bps in (4, 8, 12, 16, 17, 20, 24):
        add(f'bps{bps}', 9000, 1, bps)
    for C in (1, 2, 3, 6, 8):
        add(f'channels{C}', 5000, C, 16)
    for mode in ('independent', 'left_side', 'side_right', 'mid_side'):
        add(f'stereo_{mode}', 9000, 2, 24, stereo=mode)
    add('constant', 5000, 2, 16, pcm=np.full((5000, 2), -1234, np.int64), spec=dict(type='constant'))
    add('verbatim', 3000, 2, 16, spec=dict(type='verbatim'))
    for order in range(5):
        add(f'fixed{order}', 5000, 1, 16, spec=dict(type='fixed', order=order))
    for order, prec, shift in ((1, 2, 0), (2, 5, 3), (8, 12, None), (8, 15, 15), (12, 9, 7), (32, 15, 14), (32, 3, 1), (12, 14, 11),
                               (2, 15, 0), (8, 7, 5)):
        add(f'lpc{order}_p{prec}_s{shift}', 6000, 1, 16, spec=dict(type='lpc', order=order, precision=prec, shift=shift))
    for wasted, bps in ((1, 16), (15, 16), (23, 24), (3, 12)):
        x = speech_like(5000, 1, bps, 22050, 100 + wasted)
        x = (x >> wasted) << wasted
        add(f'wasted{wasted}_bps{bps}', 5000, 1, bps, pcm=x, spec=dict(wasted=wasted))
    add('rice', 5000, 1, 16, spec=dict(method=0))
    add('rice2', 5000, 1, 24, spec=dict(method=1))
    add('escape_raw', 5000, 1, 16, spec=dict(escape=True))
    add('escape_zero', 4096, 1, 16, pcm=np.zeros((4096, 1), np.int64), spec=dict(type='fixed', order=0, escape=True, porder=3))
    for p in range(9):
        add(f'porder{p}', 4096, 1, 16, spec=dict(type='lpc', order=8, porder=p))
    for bs in (16, 192, 576, 1000, 4096, 4608, 65535):
        add(f'block{bs}', max(3 * bs + 7, 2000), 1, 16, block_size=bs)
    add('variable', 7000, 2, 16, variable=True, blocks=[1000, 192, 4608, 1200])
    add('variable_short_last', 5000, 1, 20, variable=True, blocks=[2000, 2000, 1000])
    add('fixed_short_last', 4096 * 2 + 5, 1, 16)
    for rate in (8000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000):
        add(f'rate{rate}', 1500, 1, 16, rate=rate)
    for form, rate in (('streaminfo', 22050), ('khz', 48000), ('hz', 22050), ('tens', 44100), ('hz', 11025), ('tens', 37800)):
        add(f'rate_{form}_{rate}', 3000, 1, 16, rate=rate, header=dict(rate_form=form))
    for form in ('8', '16'):
        add(f'blockform{form}', 3000, 1, 16, block_size=192, header=dict(bs_form=form))
    add('bps_streaminfo', 3000, 1, 16, header=dict(bps_form='streaminfo'))
    return cases
