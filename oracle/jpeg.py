"""Oracle of the exact device JPEG decoder (irn_b200/csrc/jpeg_exact.cu): a numpy restatement of baseline JPEG decoding
(ITU-T T.81) with the arithmetic choices that make the result equal, bit for bit, to what libjpeg-turbo's default decompression
returns through PIL (``np.asarray(Image.open(f).convert("RGB"))``).  Pinned empirically against PIL by
tests/test_jpeg_exact_cpu.py and the fixture tests/golden/jpeg_exact.npz.

Supported streams (everything else raises JpegUnsupported; malformed or truncated headers raise JpegBadArg):
  SOF0 / SOF1, 8-bit samples, Huffman coding, one scan holding every component; 1 component (any sampling: a single-component
  scan is one block per MCU) or 3 components Y Cb Cr with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1; optional DRI.
  Progressive / lossless / arithmetic SOFs, 12-bit, 2 or 4 components, 3 components stored as RGB (Adobe transform 0, or ids
  'R','G','B' without JFIF), other samplings and DNL are unsupported.

Choices that decide the pixels:
  * Coefficients are dequantised as coef * q (integers, no clamp) in natural order (zig-zag undone at decode).
  * IDCT: the "islow" integer Loeffler-Ligtenberg-Moschytz factorisation: constants FIX(c) = round(c * 2^13) (13 fractional
    bits), pass 1 over columns keeps 2 extra bits (descale by 13 - 2 with round-half-up, x + 2^(n-1) >> n, arithmetic shift),
    pass 2 over rows descales by 13 + 2 + 3.  The result x is level-shifted through the range-limit table: x is taken modulo
    1024 into [-512, 511], then x + 128 is clamped to [0, 255].
  * Component planes are decoded padded to whole MCUs; only the first downsampled_w x downsampled_h samples of a chroma plane
    (ceil(W * h / hmax) x ceil(H * v / vmax)) take part in up-sampling.
  * Chroma up-sampling is the "fancy" triangle filter when the downsampled plane is more than 2 samples wide, plain
    replication otherwise:
      h2v1 (4:2:2): out[2c] = (3 s[c] + s[c-1] + 1) >> 2, out[2c+1] = (3 s[c] + s[c+1] + 2) >> 2; the first output column is
        s[0] and the last s[dw-1].
      h2v2 (4:2:0): per output row, the column sums t[c] = 3 s[r][c] + s[r'][c], r' = r - 1 for the upper and r + 1 for the lower
        output row of a chroma row, clamped to [0, dh - 1] (the row above the first is the first, rows below the last repeat it);
        out[2c] = (3 t[c] + t[c-1] + 8) >> 4, out[2c+1] = (3 t[c] + t[c+1] + 7) >> 4; first column (4 t[0] + 8) >> 4, last
        (4 t[dw-1] + 7) >> 4.
  * YCbCr -> RGB with 16-bit fixed point tables (FIX(x) = round(x * 2^16), half = 2^15):
      R = Y + ((FIX(1.402) (Cr-128) + half) >> 16), B = Y + ((FIX(1.772) (Cb-128) + half) >> 16),
      G = Y + ((-FIX(0.34414) (Cb-128) + half - FIX(0.71414) (Cr-128)) >> 16), each clamped to [0, 255].
  * Greyscale: R = G = B = Y.
"""
import numpy as np


class JpegUnsupported(ValueError):
    pass


class JpegBadArg(ValueError):
    pass


class JpegCorrupt(ValueError):
    pass


ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63], dtype=np.int64)   # zig-zag index -> natural (row-major) index


def _u16(d, p):
    if p + 2 > len(d):
        raise JpegBadArg("truncated header")
    return (d[p] << 8) | d[p + 1]


def parse(data):
    """Header of a supported stream: dict with H, W, nc, hs, vs (luma sampling), restart, quant [nc][64] (natural order),
    dc / ac Huffman tables per component as (counts[16], values), scan_start, scan_end (the entropy-coded bytes, EOI
    excluded).  Raises JpegUnsupported / JpegBadArg."""
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise JpegBadArg("no SOI marker")
    p = 2
    qt, dht, restart, jfif, adobe, sof = {}, {}, 0, False, None, None
    while True:
        if p >= len(d) or d[p] != 0xFF:
            raise JpegBadArg("truncated header or missing marker at byte %d" % p)
        while p < len(d) and d[p] == 0xFF:
            p += 1
        if p >= len(d):
            raise JpegBadArg("truncated header")
        m = d[p]
        p += 1
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegBadArg("unexpected marker FF%02X in the header" % m)
        L = _u16(d, p)
        if L < 2 or p + L > len(d):
            raise JpegBadArg("truncated marker segment FF%02X" % m)
        seg = d[p + 2:p + L]
        if m in (0xC0, 0xC1):
            if len(seg) < 6:
                raise JpegBadArg("short SOF")
            if seg[0] != 8:
                raise JpegUnsupported("%d-bit samples" % seg[0])
            H, W, nc = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if len(seg) < 6 + 3 * nc:
                raise JpegBadArg("short SOF")
            if H == 0:
                raise JpegUnsupported("height defined by DNL")
            if W == 0 or nc == 0:
                raise JpegBadArg("zero width or no components")
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nc)]
            sof = (H, W, nc, comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise JpegUnsupported("SOF%d (only baseline / extended sequential Huffman)" % (m - 0xC0))
        elif m == 0xCC:
            raise JpegUnsupported("arithmetic coding")
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    raise JpegBadArg("short DHT")
                tc, th = seg[q] >> 4, seg[q] & 15
                counts = list(seg[q + 1:q + 17])
                nv = sum(counts)
                if tc > 1 or th > 3 or nv > 256 or q + 17 + nv > len(seg):
                    raise JpegBadArg("bad DHT")
                code = 0
                for length in range(1, 17):       # the counts must fit the canonical code space
                    code += counts[length - 1]
                    if code > 1 << length:
                        raise JpegBadArg("bad Huffman table")
                    code <<= 1
                dht[(tc, th)] = (counts, list(seg[q + 17:q + 17 + nv]))
                q += 17 + nv
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                n = 64 * (pq + 1)
                if pq > 1 or tq > 3 or q + 1 + n > len(seg):
                    raise JpegBadArg("bad DQT")
                v = np.frombuffer(seg[q + 1:q + 1 + n], dtype=np.uint8 if pq == 0 else ">u2").astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = v
                qt[tq] = t
                q += 1 + n
        elif m == 0xDD:
            if len(seg) < 2:
                raise JpegBadArg("short DRI")
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            jfif = jfif or seg[:5] == b"JFIF\0"
        elif m == 0xEE:
            if seg[:5] == b"Adobe" and len(seg) >= 12:
                adobe = seg[11]
        elif m == 0xDC:
            raise JpegUnsupported("DNL")
        elif m == 0xDA:
            if sof is None:
                raise JpegBadArg("SOS before SOF")
            H, W, nc, comps = sof
            if len(seg) < 1 or len(seg) < 4 + 2 * seg[0]:
                raise JpegBadArg("short SOS")
            ns = seg[0]
            sc = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
            if any(c[1] > 3 or c[2] > 3 for c in sc):
                raise JpegBadArg("bad Huffman table selector")
            ss, se, a = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ns != nc or [c[0] for c in sc] != [c[0] for c in comps]:
                raise JpegUnsupported("more than one scan (non-interleaved components)")
            if ss != 0 or se != 63 or a != 0:
                raise JpegBadArg("bad spectral selection in a sequential scan")
            scan_start = p + L
            break
        p += L
    H, W, nc, comps = sof
    if nc not in (1, 3):
        raise JpegUnsupported("%d components" % nc)
    hs, vs = (1, 1) if nc == 1 else (comps[0][1], comps[0][2])
    if nc == 3:
        if (hs, vs) not in ((1, 1), (2, 1), (2, 2)) or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
            raise JpegUnsupported("sampling %s" % [(c[1], c[2]) for c in comps])
        if adobe == 0 or (adobe is None and not jfif and [c[0] for c in comps] == [82, 71, 66]):
            raise JpegUnsupported("RGB colour space")
    for c in comps:
        if c[1] < 1 or c[1] > 4 or c[2] < 1 or c[2] > 4:
            raise JpegBadArg("bad sampling factor")
    quant, dc, ac = [], [], []
    for (cid, _, _, tq), (_, td, ta) in zip(comps, sc):
        if tq not in qt or (0, td) not in dht or (1, ta) not in dht:
            raise JpegBadArg("component %d refers to a missing table" % cid)
        quant.append(qt[tq])
        dc.append(dht[(0, td)])
        ac.append(dht[(1, ta)])
    end = len(d) - 2
    while end >= scan_start and not (d[end] == 0xFF and d[end + 1] == 0xD9):
        end -= 1
    if end < scan_start:
        raise JpegBadArg("no EOI after the scan (truncated stream)")
    return dict(H=H, W=W, nc=nc, hs=hs, vs=vs, restart=restart, quant=quant, dc=dc, ac=ac, scan_start=scan_start, scan_end=end)


def inspect(data):
    """(H, W, components, h_samp, v_samp, restart_interval) of a supported stream; raises JpegUnsupported / JpegBadArg."""
    h = parse(data)
    return h["H"], h["W"], h["nc"], h["hs"], h["vs"], h["restart"]


def _huff_lookup(table):
    """{(length, code): symbol} of a canonical Huffman table (T.81 Annex C)."""
    counts, values = table
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            out[(length, code)] = values[k]
            code += 1
            k += 1
        code <<= 1
    return out


class _Bits:
    def __init__(self, data):
        self.d, self.pos, self.acc, self.n = data, 0, 0, 0

    def bit(self):
        if self.n == 0:
            if self.pos >= len(self.d):
                raise JpegCorrupt("entropy-coded segment ends early")
            self.acc, self.n = self.d[self.pos], 8
            self.pos += 1
        self.n -= 1
        return (self.acc >> self.n) & 1

    def bits(self, k):
        v = 0
        for _ in range(k):
            v = (v << 1) | self.bit()
        return v

    def symbol(self, lut):
        code = 0
        for length in range(1, 17):
            code = (code << 1) | self.bit()
            s = lut.get((length, code))
            if s is not None:
                return s
        raise JpegCorrupt("invalid Huffman code")


def _extend(v, t):
    return v - (1 << t) + 1 if t and v < (1 << (t - 1)) else v


def _segments(d):
    """Unstuffed restart intervals of an entropy-coded segment: FF 00 -> FF, split at RSTn markers."""
    segs, cur, i = [], bytearray(), 0
    while i < len(d):
        b = d[i]
        if b == 0xFF and i + 1 < len(d):
            m = d[i + 1]
            if m == 0x00:
                cur.append(0xFF)
                i += 2
                continue
            if 0xD0 <= m <= 0xD7:
                segs.append(bytes(cur))
                cur = bytearray()
                i += 2
                continue
            raise JpegCorrupt("marker FF%02X inside the scan" % m)
        cur.append(b)
        i += 1
    segs.append(bytes(cur))
    return segs


def coefficients(data, hdr=None):
    """Quantised coefficients per component: int64 [by, bx, 64] (natural order), planes padded to whole MCUs."""
    h = hdr or parse(data)
    d = bytes(data)[h["scan_start"]:h["scan_end"]]
    nc, hs, vs = h["nc"], h["hs"], h["vs"]
    mw, mh = 8 * hs, 8 * vs
    mcux, mcuy = -(-h["W"] // mw), -(-h["H"] // mh)
    samp = [(hs, vs)] + [(1, 1)] * (nc - 1)
    planes = [np.zeros((mcuy * v, mcux * hh, 64), np.int64) for hh, v in samp]
    dcl = [_huff_lookup(t) for t in h["dc"]]
    acl = [_huff_lookup(t) for t in h["ac"]]
    total = mcux * mcuy
    R = h["restart"] or total
    segs = _segments(d)
    if len(segs) < -(-total // R):
        raise JpegCorrupt("missing restart intervals")
    for k in range(-(-total // R)):
        br = _Bits(segs[k])
        pred = [0] * nc
        for m in range(k * R, min(total, (k + 1) * R)):
            my, mx = divmod(m, mcux)
            for c in range(nc):
                hh, v = samp[c]
                for by in range(v):
                    for bx in range(hh):
                        blk = planes[c][my * v + by, mx * hh + bx]
                        t = br.symbol(dcl[c])
                        if t > 15:
                            raise JpegCorrupt("bad DC category")
                        pred[c] += _extend(br.bits(t), t)
                        blk[0] = pred[c]
                        z = 1
                        while z < 64:
                            rs = br.symbol(acl[c])
                            r, s = rs >> 4, rs & 15
                            if s == 0:
                                if r != 15:
                                    break
                                z += 16
                                continue
                            z += r
                            if z > 63:
                                raise JpegCorrupt("AC run beyond the block")
                            blk[ZIGZAG[z]] = _extend(br.bits(s), s)
                            z += 1
    return planes


def _fix(x, bits):
    return int(x * (1 << bits) + 0.5)


def idct_islow(coef, q):
    """Dequantise + islow IDCT of int64 blocks [..., 64] (natural order) -> uint8 [..., 8, 8]."""
    c = (coef * q).reshape(coef.shape[:-1] + (8, 8)).astype(np.int64)
    CB = 13

    def f(x):
        return _fix(x, CB)

    def one_d(v, shift):   # v [..., 8] along the last axis
        z2, z3 = v[..., 2], v[..., 6]
        z1 = (z2 + z3) * f(0.541196100)
        tmp2 = z1 + z3 * (-f(1.847759065))
        tmp3 = z1 + z2 * f(0.765366865)
        tmp0 = (v[..., 0] + v[..., 4]) << CB
        tmp1 = (v[..., 0] - v[..., 4]) << CB
        t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
        o0, o1, o2, o3 = v[..., 7], v[..., 5], v[..., 3], v[..., 1]
        z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
        z5 = (z3 + z4) * f(1.175875602)
        o0, o1, o2, o3 = o0 * f(0.298631336), o1 * f(2.053119869), o2 * f(3.072711026), o3 * f(1.501321110)
        z1, z2 = z1 * (-f(0.899976223)), z2 * (-f(2.562915447))
        z3, z4 = z3 * (-f(1.961570560)) + z5, z4 * (-f(0.390180644)) + z5
        o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
        r = 1 << (shift - 1)
        out = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
        return np.stack([(x + r) >> shift for x in out], -1)

    ws = one_d(np.swapaxes(c, -1, -2), CB - 2)          # pass 1: columns (ws[..., col, row])
    x = one_d(np.swapaxes(ws, -1, -2), CB + 2 + 3)      # pass 2: rows
    x = ((x + 512) & 1023) - 512
    return np.clip(x + 128, 0, 255).astype(np.uint8)


def planes(data, hdr=None):
    """Sample planes (uint8 [rows, cols], padded to whole MCUs), one per component."""
    h = hdr or parse(data)
    out = []
    for c, blocks in enumerate(coefficients(data, h)):
        px = idct_islow(blocks, h["quant"][c])                       # [by, bx, 8, 8]
        out.append(px.transpose(0, 2, 1, 3).reshape(blocks.shape[0] * 8, blocks.shape[1] * 8))
    return out


def upsample(plane, H, W, hs, vs):
    """Chroma plane -> [H, W] int64 (fancy triangle filter, or replication for planes at most 2 samples wide)."""
    dw, dh = -(-W // hs), -(-H // vs)
    s = plane[:dh, :dw].astype(np.int64)
    if hs == 1 and vs == 1:
        return s[:H, :W]
    if dw <= 2:
        return np.repeat(np.repeat(s, vs, 0), hs, 1)[:H, :W]
    if vs == 2:
        up = np.concatenate([s[:1], s[:-1]], 0)       # row above, the first row repeated
        dn = np.concatenate([s[1:], s[-1:]], 0)       # row below, the last row repeated
        t = np.empty((2 * dh, dw), np.int64)
        t[0::2] = 3 * s + up
        t[1::2] = 3 * s + dn
        k, bias_even, bias_odd = 4, 8, 7
    else:
        t = s
        k, bias_even, bias_odd = 2, 1, 2
    left = np.concatenate([t[:, :1], t[:, :-1]], 1)
    right = np.concatenate([t[:, 1:], t[:, -1:]], 1)
    out = np.empty((t.shape[0], 2 * dw), np.int64)
    out[:, 0::2] = (3 * t + left + bias_even) >> k
    out[:, 1::2] = (3 * t + right + bias_odd) >> k     # at the edges the neighbour is the edge sample itself
    return out[:H, :W]


def ycc_to_rgb(y, cb, cr):
    cb, cr = cb - 128, cr - 128
    half = 1 << 15
    r = y + ((_fix(1.40200, 16) * cr + half) >> 16)
    g = y + ((-_fix(0.34414, 16) * cb + half - _fix(0.71414, 16) * cr) >> 16)
    b = y + ((_fix(1.77200, 16) * cb + half) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data):
    """uint8 [H, W, 3] RGB, equal to np.asarray(Image.open(f).convert("RGB")) for a supported stream."""
    h = parse(data)
    H, W = h["H"], h["W"]
    p = planes(data, h)
    y = p[0][:H, :W].astype(np.int64)
    if h["nc"] == 1:
        return np.repeat(y[..., None], 3, -1).astype(np.uint8)
    cb = upsample(p[1], H, W, h["hs"], h["vs"])
    cr = upsample(p[2], H, W, h["hs"], h["vs"])
    return ycc_to_rgb(y, cb, cr)
