"""CPU tests of the trajectory picture's oracle (tests/trajectory_view.py) and of the PNG writer save_trajectory() uses:
the primitive lists against the calls render_trajectory made in the unmodified reference
(tests/golden/maze_trajectory_golden.npz), the width-3 line rule, and a PNG round trip through a decoder written here."""
import os
import struct
import zlib

import numpy as np
import pytest

from oracle import maze_godview as gv
import trajectory_view as tv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "maze_trajectory_golden.npz")


def _load_cases():
    z = np.load(GOLDEN)
    out = []
    for name in z["cases"]:
        name = str(name)
        d = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + ".")}
        d["name"] = name
        out.append(d)
    return out


CASES = _load_cases()


def recorded(d, f):
    """The primitives the reference drew at recorded frame f."""
    o = d["prim_off"]
    return gv.decode(d["prims"][o[f]:o[f + 1]])


def path_at(d, f):
    o = d["traj_off"]
    return d["traj"][o[f]:o[f + 1]]


def oracle_prims(d, f):
    kind, tt, n, S, _ = (int(v) for v in d["meta"])
    task_type = ("SURVIVAL", "ESCAPE")[tt]
    return tv.trajectory_primitives(task_type, d["task.walls"], d["task.scalars"][2:4].astype(int), S, d["grid"][f][:2],
                                    [tuple(int(v) for v in p) for p in path_at(d, f)], d["food_now"][f])


def _norm(prims):
    return [(op, s, tuple(int(v) for v in c), tuple(float(v) for v in co), int(w)) for op, s, c, co, w in prims]


@pytest.mark.parametrize("d", CASES, ids=[d["name"] for d in CASES])
def test_primitives_equal_the_reference_calls(d):
    """trajectory_primitives == the reference's render_trajectory calls, call for call and bit for bit, at every frame."""
    for f in range(len(d["frames"])):
        want = _norm(recorded(d, f))
        got = _norm(oracle_prims(d, f))
        assert len(got) == len(want), (d["name"], f)
        for i, (a, b) in enumerate(zip(got, want)):
            assert a == b, (d["name"], f, i, a, b)


def test_fixture_covers_revisits_done_and_the_additional_case():
    assert len(CASES) == 36
    assert sum(int(d["done"]) for d in CASES) >= 6
    def returns(p):                                       # the agent comes back to a cell it has left
        cells = [tuple(c) for c in p.tolist()]
        runs = [c for i, c in enumerate(cells) if i == 0 or c != cells[i - 1]]
        return len(runs) > len(set(runs))
    for kind in (0, 1, 2):
        assert any(returns(path_at(d, len(d["frames"]) - 1)) for d in CASES if int(d["meta"][0]) == kind), kind
    add = [d for d in CASES if "add.names" in d]
    assert len(add) == 1
    d = add[0]
    S = int(d["meta"][3])
    aw, ah = (int(v) for v in d["add.sizes"][0])
    assert tuple(d["add.canvas"]) == (S + aw, max(S, ah))
    assert [str(v) for v in d["add.names"]] == ["traj_a.png", "traj_b.png"]
    assert d["add.blits"].tolist() == [[S, 0] + list(s) for s in d["add.sizes"].tolist()]


def test_wide_lines():
    """Width-3 rule: each Bresenham pixel becomes a 3-pixel span across the minor axis (along x when |dx| <= |dy|)."""
    horiz = set(tv.wide_line(2, 5, 6, 5))
    assert horiz == {(x, y) for x in range(2, 7) for y in (4, 5, 6)}
    vert = set(tv.wide_line(3, 9, 3, 4))
    assert vert == {(x, y) for x in (2, 3, 4) for y in range(4, 10)}
    diag = set(tv.wide_line(0, 0, 3, 3))                  # |dx| == |dy|: spans along x
    assert diag == {(i + k, i) for i in range(4) for k in (-1, 0, 1)}
    steep = set(tv.wide_line(0, 0, 1, 4))                 # y-major: the width-1 pixels widened along x
    assert steep == {(px + k, py) for px, py in gv._bresenham(0, 0, 1, 4) for k in (-1, 0, 1)}
    shallow = set(tv.wide_line(0, 0, 4, -1))              # x-major: widened along y
    assert shallow == {(px, py + k) for px, py in gv._bresenham(0, 0, 4, -1) for k in (-1, 0, 1)}
    assert set(tv.wide_line(7, 7, 7, 7)) == {(6, 7), (7, 7), (8, 7)}   # zero length: one span


def test_rasterise_draws_lines_last_and_clips():
    S = 10
    prims = [("fill", "god", (255, 255, 255), (), 0), ("rect", "god", (0, 0, 0), (0.0, 0.0, 10.0, 2.0), 0),
             ("line", "god", (255, 0, 0), (0.7, 1.2, 9.9, 1.2), 3), ("line", "god", (255, 0, 0), (0.0, 5.0, 0.0, 5.0), 3)]
    img = tv.rasterise(prims, S)
    red = (img == np.array([255, 0, 0], np.uint8)).all(-1)
    want = np.zeros((S, S), bool)
    want[0:3, 0:10] = True                                 # rows 0..2 (y - 1 clipped at the top edge is row 0)
    want[5, 0:2] = True                                    # the zero-length span at x = -1, 0, 1 clipped to 0, 1
    assert np.array_equal(red, want)
    assert (img[3:5] == 255).all() and (img[6:] == 255).all()
    with pytest.raises(AssertionError):
        tv.rasterise(prims[:2] + prims[2:3] + prims[1:2], S)


def _decode_png(data):
    """Minimal PNG reader for 8-bit RGB images with any of the five row filters."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, hdr = 8, b"", None
    while pos < len(data):
        n, tag = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xFFFFFFFF
        if tag == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        pos += 12 + n
    w, h, depth, ctype = hdr[:4]
    assert depth == 8 and ctype == 2
    raw = zlib.decompress(idat)
    stride = 3 * w
    img = np.zeros((h, stride), np.int64)
    for y in range(h):
        ft = raw[y * (stride + 1)]
        row = np.frombuffer(raw[y * (stride + 1) + 1:(y + 1) * (stride + 1)], np.uint8).astype(np.int64)
        prev = img[y - 1] if y else np.zeros(stride, np.int64)
        out = np.zeros(stride, np.int64)
        for i in range(stride):
            a = out[i - 3] if i >= 3 else 0
            b, c = prev[i], (prev[i - 3] if i >= 3 else 0)
            pred = (0, a, b, (a + b) // 2)[ft] if ft < 4 else \
                min((a, b, c), key=lambda v: (abs(a + b - c - v), (a, b, c).index(v)))
            out[i] = (row[i] + pred) & 0xFF
        img[y] = out
    return img.reshape(h, w, 3).astype(np.uint8)


@pytest.mark.parametrize("shape", [(1, 1), (7, 13), (40, 3), (64, 64)])
def test_png_round_trip(shape, tmp_path):
    from metagym_b200.png import encode_png, write_png
    rng = np.random.RandomState(shape[0] * 100 + shape[1])
    img = rng.randint(0, 256, shape + (3,)).astype(np.uint8)
    assert np.array_equal(_decode_png(encode_png(img)), img)
    p = str(tmp_path / "x.png")
    write_png(p, img)
    assert np.array_equal(_decode_png(open(p, "rb").read()), img)
    with pytest.raises(ValueError):
        encode_png(img[..., :2])
