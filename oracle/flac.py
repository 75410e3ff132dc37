"""FLAC (RFC 9639) in integer Python: the decoder csrc/flac.cu is checked against, and a test encoder that emits each coding option
on request, so that the tests reach every decoder branch whatever a real encoder would choose.

Decoder: ``parse_metadata`` (the ``fLaC`` marker, STREAMINFO, the other block types skipped), ``parse_frame_header`` (sync, codes and
tails, UTF-8 coded number, CRC-8), ``decode`` (CONSTANT / VERBATIM / FIXED 0-4 / LPC 1-32 subframes with wasted bits, Rice and Rice2
residuals with escapes, the three stereo decorrelations, CRC-16 of every frame, optionally the STREAMINFO MD5) and ``to_float``, the
conversion ``utils.audio.read_wav`` applies to a WAV file holding the same PCM.

Encoder: ``encode(pcm, sr, bps, **options)``; ``options`` are listed on ``encode``.  No float touches the coded values: the LPC
coefficients are quantised once, after which prediction and residuals are integer arithmetic."""
import hashlib

import numpy as np

BLOCK_SIZES = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, 8: 256, 9: 512, 10: 1024, 11: 2048, 12: 4096, 13: 8192, 14: 16384,
               15: 32768}
SAMPLE_RATES = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000, 11: 96000}
SAMPLE_SIZES = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
INDEPENDENT, LEFT_SIDE, SIDE_RIGHT, MID_SIDE = 'independent', 'left_side', 'side_right', 'mid_side'
META_NAMES = {0: 'STREAMINFO', 1: 'PADDING', 2: 'APPLICATION', 3: 'SEEKTABLE', 4: 'VORBIS_COMMENT', 5: 'CUESHEET', 6: 'PICTURE'}
FIXED_COEFS = ((), (1,), (2, -1), (3, -3, 1), (4, -6, 4, -1))


class FlacError(ValueError):
    """A stream that is not valid FLAC, with the byte offset where decoding stopped."""


def _crc_table(poly, width):
    top, mask, tab = 1 << (width - 1), (1 << width) - 1, []
    for b in range(256):
        c = b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        tab.append(c & mask)
    return tab


_CRC8, _CRC16 = _crc_table(0x07, 8), _crc_table(0x8005, 16)


def crc8(data):
    c = 0
    for b in data:
        c = _CRC8[c ^ b]
    return c


def crc16(data):
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


# ---------------------------------------------------------------------------------------------------------------- bit I/O
class BitReader:
    """MSB-first reader over buf[start:end] that refuses to read past ``end``."""

    def __init__(self, buf, start, end):
        self.buf, self.pos, self.end = buf, start * 8, end * 8

    def read(self, n):
        if n == 0:
            return 0
        p, e = self.pos, self.pos + n
        if e > self.end:
            raise FlacError(f'read past the end of the frame at byte {p >> 3}')
        b0, b1 = p >> 3, (e + 7) >> 3
        v = int.from_bytes(self.buf[b0:b1], 'big') >> (b1 * 8 - e)
        self.pos = e
        return v & ((1 << n) - 1)

    def signed(self, n):
        v = self.read(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self):
        n = 0
        while True:
            if self.pos >= self.end:
                raise FlacError(f'unary code runs past the end of the frame at byte {self.pos >> 3}')
            b = (self.buf[self.pos >> 3] << (self.pos & 7)) & 0xFF
            if b == 0:
                step = 8 - (self.pos & 7)
                n, self.pos = n + step, self.pos + step
                continue
            z = 8 - b.bit_length()
            self.pos += z + 1
            if self.pos > self.end:
                raise FlacError(f'unary code runs past the end of the frame at byte {self.pos >> 3}')
            return n + z

    def align(self):
        self.pos = (self.pos + 7) & ~7


class BitWriter:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def write(self, v, n):
        if n == 0:
            return
        assert 0 <= v < (1 << n), (v, n)
        self.acc, self.n = (self.acc << n) | v, self.n + n
        if self.n >= 64:
            k = self.n // 8
            self.out += (self.acc >> (self.n - 8 * k)).to_bytes(k, 'big')
            self.n -= 8 * k
            self.acc &= (1 << self.n) - 1

    def signed(self, v, n):
        assert -(1 << (n - 1)) <= v < (1 << (n - 1)), (v, n)
        self.write(v & ((1 << n) - 1), n)

    def unary(self, q):
        for _ in range(q // 32):
            self.write(0, 32)
        self.write(1, q % 32 + 1)

    def align(self):
        if self.n % 8:
            self.write(0, 8 - self.n % 8)

    def bytes(self):
        self.align()
        return bytes(self.out) + (self.acc.to_bytes(self.n // 8, 'big') if self.n else b'')


# ---------------------------------------------------------------------------------------------------------------- metadata
def parse_metadata(data, name='stream'):
    """-> (streaminfo dict, [(block type, length)], offset of the first frame).  STREAMINFO must come first; PADDING, APPLICATION,
    SEEKTABLE, VORBIS_COMMENT, CUESHEET, PICTURE and reserved types are skipped."""
    data = bytes(data)
    if data[:4] == b'OggS':
        raise FlacError(f'{name}: Ogg-encapsulated FLAC is not supported; store the stream as native FLAC (.flac)')
    if data[:4] != b'fLaC':
        raise FlacError(f'{name}: no fLaC marker at byte 0')
    off, blocks, si = 4, [], None
    while True:
        if off + 4 > len(data):
            raise FlacError(f'{name}: metadata block header runs past the end of the file at byte {off}')
        last, btype, n = data[off] >> 7, data[off] & 0x7F, int.from_bytes(data[off + 1:off + 4], 'big')
        body = data[off + 4:off + 4 + n]
        if len(body) < n or btype == 127:
            raise FlacError(f'{name}: bad metadata block (type {btype}, {n} bytes) at byte {off}')
        if (btype == 0) != (si is None):
            raise FlacError(f'{name}: STREAMINFO must be the first metadata block and appear once (byte {off})')
        if btype == 0:
            if n != 34:
                raise FlacError(f'{name}: STREAMINFO of {n} bytes at byte {off}')
            v = int.from_bytes(body[10:18], 'big')
            si = dict(min_block=int.from_bytes(body[0:2], 'big'), max_block=int.from_bytes(body[2:4], 'big'),
                      min_frame=int.from_bytes(body[4:7], 'big'), max_frame=int.from_bytes(body[7:10], 'big'),
                      sample_rate=v >> 44, channels=((v >> 41) & 7) + 1, bits=((v >> 36) & 31) + 1, total_samples=v & ((1 << 36) - 1),
                      md5=body[18:34])
        blocks.append((btype, n))
        off += 4 + n
        if last:
            return si, blocks, off


# ---------------------------------------------------------------------------------------------------------------- frames
def parse_frame_header(buf, off, end=None):
    """The frame header at byte ``off``, or None when the bytes there are not a valid header (sync code, reserved codes, the coded
    number, CRC-8).  -> dict(variable, block_size, sample_rate (0 = STREAMINFO's), channels, assignment, bits (0 = STREAMINFO's),
    number, header_bytes)."""
    end = len(buf) if end is None else end
    if off + 6 > end or buf[off] != 0xFF or (buf[off + 1] & 0xFE) != 0xF8:
        return None
    variable = buf[off + 1] & 1
    bs_code, sr_code = buf[off + 2] >> 4, buf[off + 2] & 15
    ch_code, ss_code, reserved = buf[off + 3] >> 4, (buf[off + 3] >> 1) & 7, buf[off + 3] & 1
    if bs_code == 0 or sr_code == 15 or ch_code > 10 or ss_code == 3 or reserved:
        return None
    p, b = off + 4, buf[off + 4]
    if b < 0x80:
        extra, num = 0, b
    elif 0xC0 <= b < 0xFE:
        extra = 1
        while b & (0x40 >> extra):
            extra += 1
        num = b & (0x3F >> extra)
    else:
        return None
    if extra > (6 if variable else 5) or p + 1 + extra > end:
        return None
    for i in range(extra):
        c = buf[p + 1 + i]
        if c & 0xC0 != 0x80:
            return None
        num = (num << 6) | (c & 0x3F)
    p += 1 + extra
    if bs_code in (6, 7):
        n = bs_code - 5
        if p + n > end:
            return None
        bs, p = int.from_bytes(buf[p:p + n], 'big') + 1, p + n
    else:
        bs = BLOCK_SIZES[bs_code]
    if sr_code in (12, 13, 14):
        n = 1 if sr_code == 12 else 2
        if p + n > end:
            return None
        v, p = int.from_bytes(buf[p:p + n], 'big'), p + n
        sr = v * 1000 if sr_code == 12 else v if sr_code == 13 else v * 10
    else:
        sr = SAMPLE_RATES.get(sr_code, 0)
    if p + 1 > end or crc8(buf[off:p]) != buf[p]:
        return None
    assignment = INDEPENDENT if ch_code < 8 else (LEFT_SIDE, SIDE_RIGHT, MID_SIDE)[ch_code - 8]
    return dict(variable=variable, block_size=bs, sample_rate=sr, channels=ch_code + 1 if ch_code < 8 else 2, assignment=assignment,
                bits=SAMPLE_SIZES.get(ss_code, 0), number=num, header_bytes=p + 1 - off)


def _residual(r, bs, order, pos):
    method = r.read(2)
    if method > 1:
        raise FlacError(f'reserved residual coding method {method} at byte {pos}')
    pbits, escape = (4, 15) if method == 0 else (5, 31)
    porder = r.read(4)
    if bs % (1 << porder) or (bs >> porder) < order:
        raise FlacError(f'partition order {porder} does not fit a block of {bs} at predictor order {order} (byte {pos})')
    out = []
    for part in range(1 << porder):
        n = (bs >> porder) - (order if part == 0 else 0)
        k = r.read(pbits)
        if k == escape:
            nb = r.read(5)
            out += [r.signed(nb) for _ in range(n)]
        else:
            for _ in range(n):
                u = (r.unary() << k) | r.read(k)
                out.append((u >> 1) ^ -(u & 1))
    return out


def _subframe(r, bs, bits, pos):
    if r.read(1):
        raise FlacError(f'subframe padding bit set at byte {pos}')
    t = r.read(6)
    wasted = r.unary() + 1 if r.read(1) else 0
    if wasted >= bits:
        raise FlacError(f'{wasted} wasted bits of a {bits}-bit subframe at byte {pos}')
    bits -= wasted
    if t == 0:
        x = [r.signed(bits)] * bs
    elif t == 1:
        x = [r.signed(bits) for _ in range(bs)]
    elif 8 <= t <= 12 or 32 <= t:
        order = t - 8 if t <= 12 else t - 31
        if order > bs:
            raise FlacError(f'predictor order {order} over a block of {bs} at byte {pos}')
        x = [r.signed(bits) for _ in range(order)]
        if t <= 12:
            coefs, shift = FIXED_COEFS[order], 0
        else:
            prec = r.read(4) + 1
            if prec == 16:
                raise FlacError(f'LPC precision code 15 at byte {pos}')
            shift = r.signed(5)
            if shift < 0:
                raise FlacError(f'negative LPC shift at byte {pos}')
            coefs = [r.signed(prec) for _ in range(order)]
        res = _residual(r, bs, order, pos)
        for i in range(order, bs):
            x.append(res[i - order] + (sum(c * x[i - 1 - j] for j, c in enumerate(coefs)) >> shift))
    else:
        raise FlacError(f'reserved subframe type {t} at byte {pos}')
    return [v << wasted for v in x] if wasted else x


def decode(data, name='stream', check_md5=False):
    """-> (int64 PCM [total_samples, channels], streaminfo).  Every frame's CRC-8 and CRC-16 are checked, and that the frames
    follow one another (numbers), agree with STREAMINFO and cover exactly its total; ``check_md5`` also checks the PCM's MD5."""
    data = bytes(data)
    si, _, off = parse_metadata(data, name)
    if si['total_samples'] == 0:
        raise FlacError(f'{name}: STREAMINFO gives no total sample count')
    chans, total, out, done, k = si['channels'], si['total_samples'], [], 0, 0
    while done < total:
        h = parse_frame_header(data, off)
        if h is None:
            raise FlacError(f'{name}: no valid frame header at byte {off} after {done} of {total} samples')
        want = done if h['variable'] else k
        if h['number'] != want or h['channels'] != chans or h['bits'] not in (0, si['bits']) \
                or h['sample_rate'] not in (0, si['sample_rate']) or done + h['block_size'] > total:
            raise FlacError(f'{name}: frame at byte {off} does not continue the stream or disagrees with STREAMINFO')
        r = BitReader(data, off + h['header_bytes'], len(data))
        bs, bits, sub = h['block_size'], si['bits'], []
        for c in range(chans):
            side = (h['assignment'] == LEFT_SIDE and c == 1) or (h['assignment'] == SIDE_RIGHT and c == 0) \
                or (h['assignment'] == MID_SIDE and c == 1)
            sub.append(_subframe(r, bs, bits + side, off))
        r.align()
        end = r.pos >> 3
        if end + 2 > len(data) or crc16(data[off:end + 2]) != 0:
            raise FlacError(f'{name}: CRC-16 mismatch in the frame at byte {off}')
        a, b = sub[0], sub[1] if chans > 1 else None
        if h['assignment'] == LEFT_SIDE:
            sub[1] = [x - y for x, y in zip(a, b)]
        elif h['assignment'] == SIDE_RIGHT:
            sub[0] = [x + y for x, y in zip(a, b)]
        elif h['assignment'] == MID_SIDE:
            m = [(x << 1) | (y & 1) for x, y in zip(a, b)]
            sub[0], sub[1] = [(x + y) >> 1 for x, y in zip(m, b)], [(x - y) >> 1 for x, y in zip(m, b)]
        out.append(np.array(sub, np.int64).T.reshape(bs, chans))
        done, k, off = done + bs, k + 1, end + 2
    pcm = np.concatenate(out)
    if check_md5 and md5(pcm, si['bits']) != si['md5']:
        raise FlacError(f'{name}: MD5 of the decoded PCM does not match STREAMINFO')
    return pcm, si


def md5(pcm, bits):
    """The STREAMINFO MD5: interleaved samples, little-endian, each sign-extended to a whole number of bytes."""
    nb = (bits + 7) // 8
    le = np.ascontiguousarray(pcm, dtype='<i4').view(np.uint8).reshape(-1, 4)[:, :nb]
    return hashlib.md5(le.tobytes()).digest()


def to_float(pcm, bits):
    """float32 mono samples as utils.audio.read_wav decodes a WAV file of the same PCM: sample / 2^(bits - 1), then numpy's float32
    mean(axis=1) over the C-ordered [n, channels] array scipy returns.  That sums channels in order, except exactly 8 channels,
    which numpy's pairwise sum adds as ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7)); then it divides by the count.  (The order
    follows the memory layout: the mean of an F-ordered array would add in channel order.)"""
    x = (np.asarray(pcm, np.float64) / float(1 << (bits - 1))).astype(np.float32)
    if x.ndim == 1 or x.shape[1] == 1:
        return x.reshape(-1)
    c = [x[:, i] for i in range(x.shape[1])]
    if len(c) == 8:
        y = ((c[0] + c[1]) + (c[2] + c[3])) + ((c[4] + c[5]) + (c[6] + c[7]))
    else:
        y = c[0].copy()
        for v in c[1:]:
            y += v
    return y / np.float32(len(c))


# ---------------------------------------------------------------------------------------------------------------- test encoder
def _utf8(v):
    if v < 0x80:
        return bytes([v])
    n = 1
    while v >= (1 << (5 * n + 6)):
        n += 1
    head = (0xFF00 >> (n + 1)) & 0xFF
    out = [head | (v >> (6 * n))]
    out += [0x80 | ((v >> (6 * (n - 1 - i))) & 0x3F) for i in range(n)]
    return bytes(out)


def _rice_param(vals, limit):
    if not vals:
        return 0
    m = sum((v << 1) ^ (v >> 63) for v in vals) / len(vals)
    k = 0
    while k < limit and (1 << (k + 1)) <= m:
        k += 1
    return k


def _write_residual(w, res, bs, order, opt):
    rice2 = opt.get('rice2', False)
    pbits, escape = (5, 31) if rice2 else (4, 15)
    porder = opt.get('partition_order', 0)
    while porder and (bs % (1 << porder) or (bs >> porder) < order):      # the largest order the block allows (a short last block)
        porder -= 1
    w.write(1 if rice2 else 0, 2)
    w.write(porder, 4)
    pos = 0
    esc = opt.get('escape', False)
    for part in range(1 << porder):
        n = (bs >> porder) - (order if part == 0 else 0)
        vals = res[pos:pos + n]
        pos += n
        if esc is True or (esc and part in esc):
            nb = max((max(abs(v) for v in vals) * 2 + 1).bit_length(), 0) if vals and any(vals) else opt.get('escape_zero_bits', 0)
            w.write(escape, pbits)
            w.write(nb, 5)
            for v in vals:
                w.signed(v, nb) if nb else None
        else:
            k = opt['rice_param'] if 'rice_param' in opt else _rice_param(vals, escape - 1)
            w.write(k, pbits)
            for v in vals:
                u = (v << 1) ^ (v >> 63)
                w.unary(u >> k)
                w.write(u & ((1 << k) - 1), k)


def _lpc_coefs(x, order, prec, shift):
    """Quantised least-squares predictor: any integer coefficients decode exactly, these just keep residuals small."""
    a = np.asarray(x, np.float64)
    if len(a) <= order * 2 or not np.any(a):
        c = np.zeros(order)
        c[0] = 1.0
    else:
        A = np.stack([a[order - 1 - j:len(a) - 1 - j] for j in range(order)], 1)
        c = np.linalg.lstsq(A, a[order:], rcond=None)[0]
    lim = (1 << (prec - 1)) - 1
    return [int(v) for v in np.clip(np.round(c * (1 << shift)), -lim - 1, lim)]


def _write_subframe(w, x, bits, opt):
    kind = opt.get('type', 'fixed')
    wasted = opt.get('wasted', 'auto')
    if wasted == 'auto':
        nz = [v for v in x if v]
        wasted = min(((v & -v).bit_length() - 1) for v in nz) if nz else 0
        wasted = min(wasted, bits - 1)
    x = [v >> wasted for v in x]
    bits -= wasted
    if kind == 'constant':
        assert len(set(x)) == 1, 'a CONSTANT subframe needs a constant channel'
        t = 0
    elif kind == 'verbatim':
        t = 1
    elif kind == 'fixed':
        order = opt.get('order', 2)
        t = 8 + order
    elif kind == 'lpc':
        order = opt.get('order', 8)
        t = 31 + order
    else:
        raise ValueError(kind)
    w.write(0, 1)
    w.write(t, 6)
    if wasted:
        w.write(1, 1)
        w.unary(wasted - 1)
    else:
        w.write(0, 1)
    if t == 0:
        w.signed(x[0], bits)
        return
    if t == 1:
        for v in x:
            w.signed(v, bits)
        return
    for v in x[:order]:
        w.signed(v, bits)
    if t <= 12:
        coefs, shift = FIXED_COEFS[order], 0
    else:
        prec, shift = opt.get('precision', 15), opt.get('shift', 12)
        coefs = opt['coefs'] if 'coefs' in opt else _lpc_coefs(x, order, prec, shift)
        w.write(prec - 1, 4)
        w.signed(shift, 5)
        for c in coefs:
            w.signed(c, prec)
    res = [x[i] - (sum(c * x[i - 1 - j] for j, c in enumerate(coefs)) >> shift) for i in range(order, len(x))]
    assert all(-(1 << 31) <= v < (1 << 31) for v in res), 'residual beyond 32 bits'
    _write_residual(w, res, len(x), order, opt)


def _frame(pcm, first, k, sr, bits, opt, variable):
    bs, chans = pcm.shape
    mode = opt.get('channel_mode', INDEPENDENT) if chans == 2 else INDEPENDENT
    h = bytearray([0xFF, 0xF8 | variable])
    code = {v: c for c, v in BLOCK_SIZES.items()}.get(bs) if not opt.get('block_tail') else None
    tail = b''
    if code is None:
        code, tail = (6, (bs - 1).to_bytes(1, 'big')) if bs <= 256 else (7, (bs - 1).to_bytes(2, 'big'))
    rate = opt.get('rate_code', 'auto')
    sr_codes = {v: c for c, v in SAMPLE_RATES.items()}
    if rate == 'auto':
        rate = 'table' if sr in sr_codes else 'khz' if sr % 1000 == 0 and sr // 1000 < 256 else 'tens' if sr % 10 == 0 and sr > 65535 \
            else 'hz'
    rcode, rtail = {'streaminfo': (0, b''), 'table': (sr_codes.get(sr), b''), 'khz': (12, bytes([sr // 1000])),
                    'hz': (13, sr.to_bytes(2, 'big') if sr < 65536 else None), 'tens': (14, (sr // 10).to_bytes(2, 'big'))}[rate]
    h.append((code << 4) | rcode)
    ch_code = {INDEPENDENT: chans - 1, LEFT_SIDE: 8, SIDE_RIGHT: 9, MID_SIDE: 10}[mode]
    ss = 0 if opt.get('bits_code') == 'streaminfo' else {v: c for c, v in SAMPLE_SIZES.items()}.get(bits, 0)
    h.append((ch_code << 4) | (ss << 1))
    h += _utf8(first if variable else k) + tail + rtail
    h.append(crc8(h))
    cols = [[int(v) for v in pcm[:, c]] for c in range(chans)]
    widths = [bits] * chans
    if mode != INDEPENDENT:
        L, R = cols
        S = [l - r for l, r in zip(L, R)]
        if mode == LEFT_SIDE:
            cols, widths = [L, S], [bits, bits + 1]
        elif mode == SIDE_RIGHT:
            cols, widths = [S, R], [bits + 1, bits]
        else:
            cols, widths = [[(l + r) >> 1 for l, r in zip(L, R)], S], [bits, bits + 1]
    w = BitWriter()
    subs = opt.get('subframes', [{}] * chans)
    for c in range(chans):
        _write_subframe(w, cols[c], widths[c], dict(opt.get('subframe', {}), **subs[c % len(subs)]))
    body = bytes(h) + w.bytes()
    return body + crc16(body).to_bytes(2, 'big')


def encode(pcm, sr, bits, block_size=4096, variable=False, frame_options=None, metadata=(), **options):
    """int PCM [n, channels] (or [n]) -> FLAC bytes.

    ``block_size``: one size for every frame (the last one shorter), or a list of sizes in order (their sum must be n).
    ``variable``: variable blocking strategy (sample numbers in the headers) instead of fixed (frame numbers).
    ``metadata``: block types to write after STREAMINFO (1 PADDING, 2 APPLICATION, 3 SEEKTABLE, 4 VORBIS_COMMENT, 5 CUESHEET,
    6 PICTURE), with filler bodies.
    Frame options (``options`` for every frame, ``frame_options(k)`` -> dict merged over them for frame k):
      channel_mode: independent | left_side | side_right | mid_side (stereo only); block_tail: code the size in an 8/16-bit tail;
      rate_code: auto | streaminfo | table | khz | hz | tens; bits_code: 'streaminfo' to code the sample size as 0;
      subframe: dict for every channel, subframes: list of dicts per channel, each with
        type: constant | verbatim | fixed | lpc; order; precision, shift, coefs (lpc); wasted: 'auto' or a count;
        partition_order; rice2; escape: True or a collection of partition indices; rice_param (fixed parameter)."""
    pcm = np.asarray(pcm, np.int64)
    if pcm.ndim == 1:
        pcm = pcm[:, None]
    n, chans = pcm.shape
    assert 1 <= chans <= 8 and 4 <= bits <= 32 and n > 0
    assert pcm.min() >= -(1 << (bits - 1)) and pcm.max() < (1 << (bits - 1))
    sizes = list(block_size) if not np.isscalar(block_size) else [min(block_size, n - i) for i in range(0, n, block_size)]
    assert sum(sizes) == n
    if not variable:
        assert all(s == sizes[0] for s in sizes[:-1]) and sizes[-1] <= sizes[0], 'fixed blocking: equal blocks, the last not longer'
    frames, first = [], 0
    for k, bs in enumerate(sizes):
        opt = dict(options, **(frame_options(k) if frame_options else {}))
        frames.append(_frame(pcm[first:first + bs], first, k, sr, bits, opt, int(variable)))
        first += bs
    lens = [len(f) for f in frames]
    min_b, max_b = (min(sizes), max(sizes)) if variable else (sizes[0], sizes[0])
    v = (sr << 44) | ((chans - 1) << 41) | ((bits - 1) << 36) | n
    si = min_b.to_bytes(2, 'big') + max_b.to_bytes(2, 'big') + min(lens).to_bytes(3, 'big') + max(lens).to_bytes(3, 'big') \
        + v.to_bytes(8, 'big') + md5(pcm, bits)
    blocks = [(0, si)] + [(t, _filler(t)) for t in metadata]
    out = bytearray(b'fLaC')
    for i, (t, body) in enumerate(blocks):
        out.append((0x80 if i == len(blocks) - 1 else 0) | t)
        out += len(body).to_bytes(3, 'big') + body
    for f in frames:
        out += f
    return bytes(out)


def _filler(t):
    """A body for metadata type t; the decoder skips every type but STREAMINFO, so only the length framing matters.  Bodies hold
    0xFF 0xF8 pairs on purpose: a sync pattern in metadata must not be taken for a frame."""
    return {1: bytes(37), 2: b'test' + b'\xff\xf8\x69\x08\x00' * 3, 3: (0).to_bytes(8, 'big') * 2 + bytes(2),
            4: (4).to_bytes(4, 'little') + b'test' + (0).to_bytes(4, 'little'), 5: bytes(396 + 3 + 36),
            6: bytes(32) + b'\xff\xf8'}.get(t, bytes(8))
