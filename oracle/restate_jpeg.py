"""Plain numpy restatement of the baseline JPEG decode that `torchvision.io.decode_jpeg(..., mode=RGB)` performs on the
CPU (libjpeg-turbo, islow IDCT, "fancy" upsampling, integer YCbCr->RGB), written from ITU-T T.81 and the documented
libjpeg arithmetic.  It pins the arithmetic of the device decoder (yolort_b200/csrc/jpeg_decode.cu) on a machine
without a GPU.  Only the subset the device decoder takes is restated: one interleaved baseline Huffman scan, 8-bit,
gray or YCbCr with per-component sampling ratios 1x1, 2x1 and 2x2.  Huffman decoding is pure Python: use small images.
"""
import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)


class Unsupported(ValueError):
    pass


def _u16(b, i):
    return (b[i] << 8) | b[i + 1]


def parse(data: bytes) -> dict:
    """Markers up to the end of the first scan; raises Unsupported outside the restated subset."""
    b = data
    if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise Unsupported("not a JPEG file")
    i, q, huff, ri, frame, jfif, adobe = 2, {}, {}, 0, None, False, None
    while True:
        while i < len(b) and b[i] == 0xFF and i + 1 < len(b) and b[i + 1] == 0xFF:
            i += 1
        if i + 4 > len(b) or b[i] != 0xFF:
            raise Unsupported("truncated header")
        m, ln = b[i + 1], _u16(b, i + 2)
        seg = b[i + 4:i + 2 + ln]
        if m in (0xC0, 0xC1):
            prec, h, w, nf = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            if prec != 8:
                raise Unsupported("not 8-bit")
            comps = [(seg[6 + 3 * k], seg[7 + 3 * k] >> 4, seg[7 + 3 * k] & 15, seg[8 + 3 * k]) for k in range(nf)]
            frame = (h, w, comps)
        elif m == 0xC4:
            k = 0
            while k < len(seg):
                tc, th = seg[k] >> 4, seg[k] & 15
                counts = list(seg[k + 1:k + 17])
                vals = list(seg[k + 17:k + 17 + sum(counts)])
                huff[(tc, th)] = (counts, vals)
                k += 17 + sum(counts)
        elif m == 0xDB:
            k = 0
            while k < len(seg):
                pq, tq = seg[k] >> 4, seg[k] & 15
                if pq:
                    t = [_u16(seg, k + 1 + 2 * j) for j in range(64)]
                    k += 129
                else:
                    t = list(seg[k + 1:k + 65])
                    k += 65
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = t
                q[tq] = nat
        elif m == 0xDD:
            ri = _u16(seg, 0)
        elif m == 0xE0:
            jfif = jfif or (len(seg) >= 5 and bytes(seg[:5]) == b"JFIF\0")
        elif m == 0xEE:
            if len(seg) >= 12 and bytes(seg[:5]) == b"Adobe":
                adobe = seg[11]
        elif m == 0xDA:
            ns = seg[0]
            sel = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(ns)]
            start = i + 2 + ln
            break
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        else:
            raise Unsupported(f"marker 0x{m:02X}")
        i += 2 + ln
    if frame is None:
        raise Unsupported("no SOF0/SOF1 frame")
    h, w, comps = frame
    if len(comps) not in (1, 3) or len(sel) != len(comps):
        raise Unsupported("component count")
    if len(comps) == 3:
        ids = [c[0] for c in comps]
        if not jfif and (adobe == 0 or (adobe is None and ids == [82, 71, 66])):
            raise Unsupported("RGB colour space")
    return dict(h=h, w=w, comps=comps, sel=sel, q=q, huff=huff, ri=ri, start=start)


class _Bits:
    """Entropy-coded bytes with stuffing removed; RSTn markers end an interval."""

    def __init__(self, b, i):
        self.b, self.i, self.acc, self.n = b, i, 0, 0

    def bit(self):
        if self.n == 0:
            c = self.b[self.i]
            if c == 0xFF:
                nxt = self.b[self.i + 1]
                if nxt == 0:
                    self.i += 1
                else:
                    raise ValueError("hit a marker inside an interval")
            self.i += 1
            self.acc, self.n = c, 8
        self.n -= 1
        return (self.acc >> self.n) & 1

    def bits(self, s):
        v = 0
        for _ in range(s):
            v = (v << 1) | self.bit()
        return v

    def restart(self):
        self.n = 0
        while self.b[self.i] == 0xFF and self.b[self.i + 1] == 0xFF:
            self.i += 1
        if not (self.b[self.i] == 0xFF and 0xD0 <= self.b[self.i + 1] <= 0xD7):
            raise ValueError("missing restart marker")
        self.i += 2


def _table(counts, vals):
    code, k, out = 0, 0, {}
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out[(ln, code)] = vals[k]
            k += 1
            code += 1
        code <<= 1
    return out


def _decode(br, tab):
    code = 0
    for ln in range(1, 17):
        code = (code << 1) | br.bit()
        s = tab.get((ln, code))
        if s is not None:
            return s
    raise ValueError("invalid Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(info, data):
    """Quantised coefficients per component: [blocks_y, blocks_x, 64] int16, natural order."""
    h, w, comps = info["h"], info["w"], info["comps"]
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    single = len(comps) == 1
    if single:
        mx, my = -(-w // 8), -(-h // 8)
        layout = [(0, 0, 0)]
        planes = [np.zeros((my, mx, 64), np.int16)]
    else:
        mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
        layout = [(ci, v, u) for ci, c in enumerate(comps) for v in range(c[2]) for u in range(c[1])]
        planes = [np.zeros((my * c[2], mx * c[1], 64), np.int16) for c in comps]
    tabs = {k: _table(*v) for k, v in info["huff"].items()}
    sel = {s[0]: (s[1], s[2]) for s in info["sel"]}
    dct = [(tabs[(0, sel[c[0]][0])], tabs[(1, sel[c[0]][1])]) for c in comps]
    br = _Bits(data, info["start"])
    ri = info["ri"]
    pred = [0] * len(comps)
    for m in range(mx * my):
        if ri and m and m % ri == 0:
            br.restart()
            pred = [0] * len(comps)
        for ci, v, u in layout:
            dtab, atab = dct[ci]
            blk = np.zeros(64, np.int64)
            s = _decode(br, dtab)
            pred[ci] += _extend(br.bits(s), s)
            blk[0] = pred[ci]
            k = 1
            while k < 64:
                rs = _decode(br, atab)
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    if k > 63:
                        raise ValueError("coefficient index past 63")
                    blk[ZIGZAG[k]] = _extend(br.bits(s), s)
                    k += 1
                elif r == 15:
                    k += 16
                else:
                    break
            c = comps[ci]
            by, bx = (m // mx, m % mx) if single else ((m // mx) * c[2] + v, (m % mx) * c[1] + u)
            planes[ci][by, bx] = blk.astype(np.int16)       # libjpeg keeps JCOEF (16-bit) coefficients
    return planes


_F = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137,
          c1961=16069, c2053=16819, c2562=20995, c3072=25172)


def _idct_1d(x, shift):
    """One islow pass over axis -1 (8 inputs): returns the 8 outputs descaled by `shift` (int64 arithmetic)."""
    f = _F
    z2, z3 = x[..., 2], x[..., 6]
    z1 = (z2 + z3) * f["c0541"]
    tmp2 = z1 - z3 * f["c1847"]
    tmp3 = z1 + z2 * f["c0765"]
    tmp0 = (x[..., 0] + x[..., 4]) << 13
    tmp1 = (x[..., 0] - x[..., 4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * f["c1175"]
    o0, o1, o2, o3 = o0 * f["c0298"], o1 * f["c2053"], o2 * f["c3072"], o3 * f["c1501"]
    z1, z2 = z1 * -f["c0899"], z2 * -f["c2562"]
    z3, z4 = z3 * -f["c1961"] + z5, z4 * -f["c0390"] + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    r = 1 << (shift - 1)
    out = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
    return np.stack([(v + r) >> shift for v in out], axis=-1)


def idct_islow(coef, qtab):
    """[..., 64] int16 coefficients (natural order) x quant table -> [..., 8, 8] uint8 samples.  libjpeg's C code ends
    in range_limit[x & 1023]; its SIMD code saturates.  Both agree for x in [-512, 511], the only range
    `range_ok` accepts (the device decoder routes blocks outside it back to the CPU)."""
    d = coef.astype(np.int64) * qtab.astype(np.int64)
    blk = d.reshape(coef.shape[:-1] + (8, 8))
    cols = _idct_1d(np.swapaxes(blk, -1, -2), 13 - 2)           # pass 1: columns, PASS1_BITS = 2
    rows = _idct_1d(np.swapaxes(cols, -1, -2), 13 + 2 + 3)      # pass 2: rows
    return np.clip(rows + 128, 0, 255).astype(np.uint8), (d, cols, rows)


def range_ok(parts) -> bool:
    d, cols, rows = parts
    return bool(np.abs(d).max(initial=0) <= 32767 and np.abs(cols).max(initial=0) <= 32767
                and rows.min(initial=0) >= -512 and rows.max(initial=0) <= 511)


def _up_h2(p, w_ds, fancy, bias_even, bias_odd, scale):
    """Horizontal 2x of rows `p` ([rows, >= w_ds]) with the triangle filter (3a + neighbour + bias) >> scale."""
    if not fancy:
        return np.repeat(p[:, :w_ds], 2, axis=1)
    c = p[:, :w_ds].astype(np.int64)
    left = np.concatenate([c[:, :1], c[:, :-1]], axis=1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], axis=1)
    out = np.empty((p.shape[0], 2 * w_ds), np.int64)
    out[:, 0::2] = (3 * c + left + bias_even) >> scale
    out[:, 1::2] = (3 * c + right + bias_odd) >> scale
    return out


def upsample(plane, w_ds, h_ds, hr, vr):
    """libjpeg's upsamplers for ratio (hr, vr) of one component: fullsize, h2v1 fancy (+1/+2 >> 2), h2v2 fancy
    (vertical 3:1 then horizontal 3:1, +8/+7 >> 4).  Fancy only when the downsampled width exceeds 2, else box."""
    p = plane[:h_ds, :].astype(np.int64)
    fancy = w_ds > 2
    if (hr, vr) == (1, 1):
        return p[:, :w_ds]
    if (hr, vr) == (2, 1):
        return _up_h2(p, w_ds, fancy, 1, 2, 2) if fancy else np.repeat(p[:, :w_ds], 2, axis=1)
    if not fancy:
        return np.repeat(np.repeat(p[:, :w_ds], 2, axis=0), 2, axis=1)
    above = np.concatenate([p[:1], p[:-1]], axis=0)
    below = np.concatenate([p[1:], p[-1:]], axis=0)
    out = np.empty((2 * h_ds, 2 * w_ds), np.int64)
    out[0::2] = _up_h2(3 * p + above, w_ds, True, 8, 7, 4)
    out[1::2] = _up_h2(3 * p + below, w_ds, True, 8, 7, 4)
    return out


def ycc_to_rgb(y, cb, cr):
    """libjpeg's integer tables (jdcolor.c): 16 fractional bits, Cr->R and Cb->B rounded once, G summed then shifted."""
    def fix(v):
        return int(v * 65536 + 0.5)
    cb, cr = cb - 128, cr - 128
    r = y + ((fix(1.40200) * cr + 32768) >> 16)
    b = y + ((fix(1.77200) * cb + 32768) >> 16)
    g = y + ((-fix(0.34414) * cb + 32768 - fix(0.71414) * cr) >> 16)
    return np.clip(np.stack([r, g, b]), 0, 255).astype(np.uint8)


def decode(data: bytes) -> np.ndarray:
    """[3, H, W] uint8, the bytes torchvision.io.decode_jpeg(..., mode=RGB) returns for files of the subset."""
    data = bytes(data)
    info = parse(data)
    h, w, comps = info["h"], info["w"], info["comps"]
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    planes = coefficients(info, data)
    comp_px = []
    for ci, c in enumerate(comps):
        by, bx = planes[ci].shape[:2]
        px, parts = idct_islow(planes[ci], info["q"][c[3]])
        if not range_ok(parts):
            raise Unsupported("IDCT values outside the exactly reproducible range")
        img = px.transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)
        w_ds, h_ds = -(-w * c[1] // hmax), -(-h * c[2] // vmax)
        comp_px.append(upsample(img, w_ds, h_ds, hmax // c[1], vmax // c[2])[:h, :w])
    if len(comps) == 1:
        return np.repeat(comp_px[0].astype(np.uint8)[None], 3, axis=0)
    return ycc_to_rgb(*comp_px)
