"""Test helper: insert an APP1 Exif segment holding an Orientation tag (274, SHORT) right after SOI of any JPEG file.

Big- or little-endian TIFF; optionally other IFD0 entries around the tag (so it is not the first entry) and an IFD1."""
import struct


def with_orientation(jpeg, value, big_endian=True, tag_last=False, ifd1=False):
    assert jpeg[:2] == b"\xff\xd8"
    e = ">" if big_endian else "<"

    def entry(tag, typ, count, raw4):
        return struct.pack(e + "HHI", tag, typ, count) + raw4

    short = lambda v: struct.pack(e + "HH", v, 0)   # SHORT values sit left-justified in the 4-byte field
    entries = [entry(274, 3, 1, short(value))]
    if tag_last:   # other tags first (ImageWidth, ImageLength, ResolutionUnit): the parser must walk to 274
        entries = [entry(256, 4, 1, struct.pack(e + "I", 64)), entry(257, 4, 1, struct.pack(e + "I", 48))] + entries + \
                  [entry(296, 3, 1, short(2))]
    ifd0_off = 8
    ifd0_len = 2 + 12 * len(entries) + 4
    next_off = ifd0_off + ifd0_len if ifd1 else 0
    tiff = (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 42, ifd0_off)
    tiff += struct.pack(e + "H", len(entries)) + b"".join(entries) + struct.pack(e + "I", next_off)
    if ifd1:   # IFD1 with Compression = 6 and no thumbnail offset: not a thumbnail the decoder could use
        tiff += struct.pack(e + "H", 1) + entry(259, 3, 1, short(6)) + struct.pack(e + "I", 0)
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + struct.pack(">H", len(body) + 2) + body + jpeg[2:]


def transform(img, k):
    """T_k of an [rows, cols, ...] array: the EXIF transform k (PIL's exif_transpose operations)"""
    if k == 1:
        return img
    if k == 2:
        return img[:, ::-1]
    if k == 3:
        return img[::-1, ::-1]
    if k == 4:
        return img[::-1, :]
    t = img.swapaxes(0, 1)
    if k == 5:
        return t
    if k == 6:
        return t[:, ::-1]
    if k == 7:
        return img[::-1, ::-1].swapaxes(0, 1)
    if k == 8:
        return t[::-1, :]
    raise ValueError(k)
