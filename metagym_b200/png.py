"""Minimal PNG writer (8-bit RGB, no filtering) on the standard library, for save_trajectory(): the batched envs do not
depend on pygame or PIL."""
import struct
import zlib

import numpy as np

_SIGNATURE = b"\x89PNG\r\n\x1a\n"


def _chunk(tag, data):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def encode_png(rgb):
    """uint8 [H, W, 3] image, rows top to bottom -> the bytes of a PNG file."""
    img = np.ascontiguousarray(rgb, dtype=np.uint8)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError("encode_png needs a uint8 [H, W, 3] image, got shape %s" % (img.shape,))
    h, w = img.shape[:2]
    rows = np.zeros((h, 1 + 3 * w), dtype=np.uint8)          # filter byte 0 (None) ahead of every row
    rows[:, 1:] = img.reshape(h, 3 * w)
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)       # 8 bits per channel, colour type 2 (RGB)
    return _SIGNATURE + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", zlib.compress(rows.tobytes(), 6)) + _chunk(b"IEND", b"")


def write_png(file_name, rgb):
    with open(file_name, "wb") as f:
        f.write(encode_png(rgb))
