"""CPU checks of the layout helper of tests/test_large_index_gpu.py: the straddling rows it returns for fake layouts, and
that every shape of the GPU file really crosses the 32-bit boundaries it exists for (so that the claim "this test covers
byte 2^32" holds without a GPU)."""
import pytest

from util import B31, B32, E31, LARGE_SHAPES, crossings, layout_bytes, straddle_rows, twin_bases


def test_crossings_of_fake_layouts():
    assert crossings(None, 1 << 20, 2048, 4) == set()                      # exactly 2^31 bytes: last offset 2^31 - 1
    assert crossings(None, (1 << 20) + 1, 2048, 4) == {B31}
    assert crossings(2, (1 << 20) + 1, 2048, 4) == {B31, B32}
    assert crossings(2, (1 << 20) + 1, 2048, 1) == {B31, B32, E31}
    assert crossings(3, 1 << 30, 4, 2) == {B31, B32, E31}
    assert crossings(2, 1 << 30, 4, 4) == {B31, B32}                       # 2^31 elements: last index 2^31 - 1


def test_straddle_rows_hold_each_boundary():
    T, n, rb = 5, 1000003, 1000
    rows, held = straddle_rows(T, n, rb, 4, seed=3)
    assert set(held) == {B31, B32}
    for name, byte in ((B31, 1 << 31), (B32, 1 << 32)):
        t, e = held[name]
        r = t * n + e
        assert r * rb <= byte < (r + 1) * rb                                # the row holds the boundary byte
        for q in (r - 1, r, r + 1):                                         # ... and its neighbours are compared too
            assert (q // n, q % n) in rows
    for t in (0, T - 1):
        for e in (0, 1, n - 2, n - 1):
            assert (t, e) in rows
    assert rows == sorted(set(rows)) and all(0 <= t < T and 0 <= e < n for t, e in rows)
    assert len(rows) >= 8 + 6                                               # edges, boundaries, seeded extras
    assert straddle_rows(T, n, rb, 4, seed=3) == (rows, held)               # seeded: the same rows every run


def test_straddle_rows_boundary_on_a_row_edge():
    """A boundary that falls exactly between two rows: the rows on both sides are compared."""
    n, rb = (1 << 22) + 5, 1024                                            # row 2^21 starts at byte 2^31, row 2^22 at 2^32
    rows, held = straddle_rows(None, n, rb, 1)
    assert held == {B31: (0, 1 << 21), E31: (0, 1 << 21), B32: (0, 1 << 22)}
    for e in (1 << 21, 1 << 22):
        assert (0, e - 1) in rows and (0, e) in rows
    n = 1 << 22                                                             # ends exactly at byte 2^32: not crossed
    assert crossings(None, n, rb, 1) == {B31, E31}
    assert B32 not in straddle_rows(None, n, rb, 1)[1]


def test_twin_bases_cover_every_env():
    n = 1000
    envs = [0, 1, 2, 3, 500, 501, 998, 999, 700]
    bases = twin_bases(envs, n)
    assert all(0 <= b <= n - 3 for b in bases)
    assert all(any(b <= e < b + 3 for b in bases) for e in envs)
    assert bases == sorted(bases) and len(bases) == 5                       # 0..2, 2..4, 499..501, 699..701, 997..999


@pytest.mark.parametrize("name", sorted(LARGE_SHAPES))
def test_large_shapes_cross_what_they_claim(name):
    """Every output the GPU test names crosses the boundaries listed for it (element index 2^31 of 1-byte elements is
    byte 2^31)."""
    for out, T, n, rb, eb, claim in LARGE_SHAPES[name]:
        got = crossings(T, n, rb, eb)
        assert claim <= got, (name, out, layout_bytes(T, n, rb), got)
        _, held = straddle_rows(T, n, rb, eb)
        assert claim <= set(held), (name, out)


def test_large_shapes_claims():
    """The boundaries each GPU test exists for (issue table): byte 2^32 of the big rollouts and views, element 2^31 of the
    quadrotor rollout, the int32 3-D rollout, the 2-D rollout and the path record; byte 2^31 of the streamed step."""
    claim = {k: set().union(*[c for *_, c in v]) for k, v in LARGE_SHAPES.items()}
    assert claim["quad_step_stream"] == {B31}
    assert E31 in claim["quad_rollout"] and B32 in claim["quad_rollout_final"]
    for k in ("maze3d_step_u8", "maze3d_rollout_u8", "mazec3d_rollout_u8", "god_view", "path"):
        assert B32 in claim[k], k
    for k in ("maze3d_rollout_i32", "maze2d_rollout", "path"):
        assert E31 in claim[k], k
    # the path record of PATH_N envs puts element 2^31 at step 976, inside a 990-step rollout
    _, held = straddle_rows(*LARGE_SHAPES["path"][0][1:5])
    assert held[E31][0] == 976 and held[B31][0] == 488
