"""An independent statement of the project's JPEG format (TEST INFRASTRUCTURE): fp64 DCT (scipy.fft.dctn), its own quantisation, its own Huffman
tables, bit writer, byte stuffing and markers, written from ITU-T T.81 and sharing no code with uhc_b200/csrc/video_core.h.

The format: JFIF, full-range BT.601 YCbCr in 16-bit fixed point, 4:2:0 (the chroma sample is the rounded mean of its 2 x 2 values), edges
replicated, the Annex K tables scaled as IJG does, the Annex K Huffman tables, one restart interval per MCU row."""
import numpy as np
from scipy.fft import dctn

ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56,
               57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
LUM = np.array([[16, 11, 10, 16, 24, 40, 51, 61], [12, 12, 14, 19, 26, 58, 60, 55], [14, 13, 16, 24, 40, 57, 69, 56], [14, 17, 22, 29, 51, 87, 80, 62],
                [18, 22, 37, 56, 68, 109, 103, 77], [24, 35, 55, 64, 81, 104, 113, 92], [49, 64, 78, 87, 103, 121, 120, 101],
                [72, 92, 95, 98, 112, 100, 103, 99]])
CHR = np.full((8, 8), 99)
CHR[:4, :4] = [[17, 18, 24, 47], [18, 21, 26, 66], [24, 26, 56, 99], [47, 66, 99, 99]]

# Annex K.3: (counts of codes of length 1 .. 16, symbols)
DC_LUM = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHR = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUM = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125], list(bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a434445464748494a"
    "535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7"
    "c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")))
AC_CHR = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119], list(bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738393a434445464748"
    "494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4"
    "c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")))


def huff_codes(spec):
    """symbol -> bit string of the canonical code (T.81 Annex C)"""
    counts, syms = spec
    out, code, i = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out[syms[i]] = format(code, "0%db" % ln)
            code, i = code + 1, i + 1
        code <<= 1
    return out


def quant_tables(q):
    """[2][8][8] luminance and chrominance tables of quality q (natural order)"""
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.stack([np.clip((t * s + 50) // 100, 1, 255) for t in (LUM, CHR)])


def planes(rgb):
    """rgb [H][W][3] uint8 -> Y [H16][W16], Cb, Cr [H16 / 2][W16 / 2] ints, the frame padded to whole MCUs by repeating its last row / column"""
    H, W = rgb.shape[:2]
    H16, W16 = -(-H // 16) * 16, -(-W // 16) * 16
    p = np.pad(rgb.astype(np.int64), ((0, H16 - H), (0, W16 - W), (0, 0)), mode="edge")
    r, g, b = p[..., 0], p[..., 1], p[..., 2]
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16         # a rounding term one below a half keeps Cb, Cr <= 255
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16
    sub = lambda c: (c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + 2) >> 2
    return y, sub(cb), sub(cr)


def blocks(rgb):
    """level-shifted samples [mcu rows][mcu cols][6][8][8] (Y0 Y1 Y2 Y3 Cb Cr)"""
    y, cb, cr = planes(rgb)
    my, mx = y.shape[0] // 16, y.shape[1] // 16
    out = np.zeros((my, mx, 6, 8, 8), np.int64)
    Y = y.reshape(my, 2, 8, mx, 2, 8).transpose(0, 3, 1, 4, 2, 5).reshape(my, mx, 4, 8, 8)
    out[:, :, :4] = Y
    out[:, :, 4] = cb.reshape(my, 8, mx, 8).transpose(0, 2, 1, 3)
    out[:, :, 5] = cr.reshape(my, 8, mx, 8).transpose(0, 2, 1, 3)
    return out - 128


def dct(b):
    """the orthonormal 2-D DCT-II (JPEG's FDCT) in fp64 over the last two axes"""
    return dctn(np.asarray(b, np.float64), type=2, norm="ortho", axes=(-2, -1))


def quantise(F, q):
    """F / Q rounded half away from zero, AC and DC clamped to +-1023; F [..][6][8][8] -> zigzag [..][6][64]"""
    t = quant_tables(q)
    Qb = np.stack([t[0]] * 4 + [t[1]] * 2)
    r = F / Qb
    v = np.sign(r) * np.floor(np.abs(r) + 0.5)
    v = np.clip(v, -1023, 1023).astype(np.int64)
    return v.reshape(v.shape[:-2] + (64,))[..., ZZ], (r.reshape(r.shape[:-2] + (64,))[..., ZZ])


def coefs(rgb, q):
    """(quantised coefficients [mcu rows][mcu cols][6][64] zigzag, the unrounded F / Q in the same layout)"""
    return quantise(dct(blocks(rgb)), q)


def _category(v):
    return int(abs(int(v))).bit_length()


def _extra(v, n):
    return format(v if v >= 0 else v + (1 << n) - 1, "0%db" % n) if n else ""


def entropy_segment(row):
    """one MCU row of coefficients [mcu cols][6][64] -> its bytes: Huffman coded, padded with 1-bits, 0xFF stuffed"""
    dcl, dcc, acl, acc = (huff_codes(s) for s in (DC_LUM, DC_CHR, AC_LUM, AC_CHR))
    bits = []
    pred = [0, 0, 0]
    for mcu in row:
        for b in range(6):
            comp = 0 if b < 4 else b - 3
            dc_t, ac_t = (dcl, acl) if comp == 0 else (dcc, acc)
            zz = mcu[b]
            d = int(zz[0]) - pred[comp]
            pred[comp] = int(zz[0])
            n = _category(d)
            bits.append(dc_t[n] + _extra(d, n))
            nz = np.nonzero(zz[1:])[0] + 1
            last = 0
            for k in nz:
                run = k - last - 1
                while run >= 16:
                    bits.append(ac_t[0xF0])
                    run -= 16
                n = _category(zz[k])
                bits.append(ac_t[(run << 4) | n] + _extra(int(zz[k]), n))
                last = k
            if last != 63:
                bits.append(ac_t[0x00])
    s = "".join(bits)
    s += "1" * (-len(s) % 8)
    raw = np.packbits(np.frombuffer(s.encode(), np.uint8) - 48).tobytes() if s else b""
    return raw.replace(b"\xff", b"\xff\x00")


def _seg(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def header(W, H, q):
    t = quant_tables(q)
    h = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for c in range(2):
        h += _seg(0xDB, bytes([c]) + bytes(int(x) for x in t[c].reshape(64)[ZZ]))
    h += _seg(0xC0, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for cls, spec in ((0x00, DC_LUM), (0x10, AC_LUM), (0x01, DC_CHR), (0x11, AC_CHR)):
        h += _seg(0xC4, bytes([cls]) + bytes(spec[0]) + bytes(spec[1]))
    h += _seg(0xDD, (-(-W // 16)).to_bytes(2, "big"))
    h += _seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    return h


def file_from_coefs(c, W, H, q):
    """a JPEG file from quantised coefficients [mcu rows][mcu cols][6][64] (zigzag)"""
    out = header(W, H, q)
    for r, row in enumerate(c):
        if r:
            out += bytes([0xFF, 0xD0 + ((r - 1) & 7)])
        out += entropy_segment(row)
    return out + b"\xff\xd9"


def encode(rgb, q):
    """one frame rgb [H][W][3] uint8 -> a JPEG file (bytes) through the fp64 DCT"""
    H, W = rgb.shape[:2]
    return file_from_coefs(coefs(rgb, q)[0], W, H, q)
