"""Model check of scan3.cu's k <= 32 candidate epilogue hand-over: the scanners keep the last data buffer of a tile
(the zero stage's previous buffer) as the tile's sum area and give it back to the stagers only when every scanner warp
has finished its query.

One stager role and W scanner warps.  FULL(b) is an mbarrier per ring buffer (every scanner warp waits on the phase
parity it tracks); EMPTY(b) is a named barrier that completes when ALL scanner warps have arrived and the stager syncs;
BAR_SCAN is a named barrier of the W scanner warps.  Per tile, at the zero stage, each warp: reads the stage, syncs
BAR_SCAN, writes its rows' sums into the held buffer, syncs BAR_SCAN, runs the epilogue of its query (warp w < ng of the
tile) reading the sums, and only then arrives on EMPTY of the held buffer (when a next tile exists).  Random
interleavings check: no deadlock; the stager never rewrites a buffer that holds sums some warp has still to read; the
sums a warp reads are its own tile's; a warp never arrives twice on one EMPTY generation (a named barrier would complete
without the stager); a FULL phase is never completed twice before every warp consumed it; scanner warps drift apart by
at most two stages."""
import random

import pytest


def ring_next(b):
    return 0 if b == 2 else b + 1


def stager(ng_of_tiles, nch, st, W):
    b = gs = 0
    for _ in ng_of_tiles:
        for _ch in range(nch + 1):
            if gs >= 2:
                while st["empty_arrivals"][b] < W:           # bar.sync EMPTY(b): needs every scanner warp
                    yield "blocked"
                st["empty_arrivals"][b] -= W
                st["empty_pending"][b] = [False] * W
            assert st["readers"][b] == 0, f"buffer {b} rewritten while read (stage {gs})"
            assert st["holders"][b] == 0, f"buffer {b} rewritten while it holds sums still to be read (stage {gs})"
            assert all(c >= st["full_done"][b] for c in st["consumed"][b]), f"FULL({b}) phase would alias at stage {gs}"
            st["stage"][b] = gs
            st["sums"][b] = None
            st["full_done"][b] += 1
            yield "progress"
            b = ring_next(b)
            gs += 1


def scan_barrier(st, w, W):
    """bar.sync BAR_SCAN over the W scanner warps."""
    gen = st["bar_gen"]
    st["bar_count"] += 1
    if st["bar_count"] == W:
        st["bar_count"] = 0
        st["bar_gen"] += 1
    while st["bar_gen"] == gen:
        yield "blocked"


def arrive_empty(st, w, b):
    assert not st["empty_pending"][b][w], f"warp {w} arrived twice on one EMPTY({b}) generation"
    st["empty_pending"][b][w] = True
    st["empty_arrivals"][b] += 1


def scanner(w, ng_of_tiles, nch, st, W, rng):
    b = gs = 0
    ph = 0
    ntiles = len(ng_of_tiles)
    for n, ng in enumerate(ng_of_tiles):
        next_exists = n + 1 < ntiles
        for it in range(nch + 1):
            while not st["full_done"][b] > st["consumed"][b][w]:   # mbarrier.try_wait.parity
                yield "blocked"
            assert (st["consumed"][b][w] & 1) == ((ph >> b) & 1), "parity mask out of step with the phases consumed"
            st["consumed"][b][w] += 1
            ph ^= 1 << b
            bp = 2 if b == 0 else b - 1
            assert st["stage"][b] == gs, f"warp {w} stage {gs}: buffer {b} holds {st['stage'][b]}"
            assert st["stage"][bp] == gs - 1, f"warp {w} stage {gs}: previous buffer holds {st['stage'][bp]}"
            st["pos"][w] = gs
            live = [p for p in st["pos"] if p < (1 << 30)]
            assert max(live) - min(live) <= 2, f"scanner warps drifted {st['pos']}"
            st["readers"][b] += 1; st["readers"][bp] += 1
            yield "progress"
            st["readers"][b] -= 1; st["readers"][bp] -= 1
            if it < nch:
                if it + 2 <= nch or next_exists:
                    arrive_empty(st, w, bp)
                    yield "progress"
            else:
                # candidate epilogue: bp (the last data buffer) becomes the tile's sum area
                yield from scan_barrier(st, w, W)
                assert st["readers"][bp] == 0, "sums written while a warp still reads the last data buffer"
                assert st["stage"][bp] == gs - 1, "last data buffer rewritten before its sums were written"
                st["sums"][bp] = n
                st["holders"][bp] += 1
                yield "progress"
                yield from scan_barrier(st, w, W)
                if w < ng:                                    # warp w runs query w of the tile
                    for _ in range(rng.randint(1, 4)):        # stats, bisection and append passes
                        assert st["sums"][bp] == n and st["stage"][bp] == gs - 1, \
                            f"warp {w} tile {n}: sums overwritten"
                        yield "progress"
                st["holders"][bp] -= 1
                if next_exists:
                    arrive_empty(st, w, bp)
                    yield "progress"
            b = ring_next(b)
            gs += 1
    st["pos"][w] = 1 << 30                                    # done: no longer bounds the drift


def run(ng_of_tiles, nch, W, seed):
    rng = random.Random(seed)
    st = {"stage": {0: None, 1: None, 2: -1}, "readers": {0: 0, 1: 0, 2: 0}, "holders": {0: 0, 1: 0, 2: 0},
          "sums": {0: None, 1: None, 2: None}, "full_done": {0: 0, 1: 0, 2: 0},
          "consumed": {b: [0] * W for b in range(3)}, "empty_arrivals": {0: 0, 1: 0, 2: 0},
          "empty_pending": {b: [False] * W for b in range(3)}, "pos": [0] * W, "bar_count": 0, "bar_gen": 0}
    roles = {"S": stager(ng_of_tiles, nch, st, W)}
    roles.update({f"C{w}": scanner(w, ng_of_tiles, nch, st, W, rng) for w in range(W)})
    live = set(roles)
    blocked = set()                                           # roles that made no progress since the last progress
    while live:
        r = rng.choice(sorted(live))
        try:
            ev = next(roles[r])
        except StopIteration:
            live.discard(r)
            blocked.clear()
            continue
        if ev == "blocked":
            blocked.add(r)
            assert blocked != live, f"deadlock: {sorted(live)} all wait"
        else:
            blocked.clear()
    assert all(v == 0 for v in st["readers"].values())
    assert all(v == 0 for v in st["holders"].values())


@pytest.mark.parametrize("nch", [1, 2, 3, 12])
@pytest.mark.parametrize("W", [1, 2, 8])
def test_epilogue_hold_any_tile_length(nch, W):
    for ntiles in (1, 2, 5):
        for seed in range(6):
            run([W] * ntiles, nch, W, seed)


@pytest.mark.parametrize("nch", [1, 2, 12])
def test_epilogue_hold_varying_ng(nch):
    """Consecutive tiles with different query counts, so some warps have no query and go straight on."""
    for seed in range(24):
        rng = random.Random(1000 + seed)
        ng_of_tiles = [rng.randint(1, 8) for _ in range(rng.randint(1, 7))]
        run(ng_of_tiles, nch, 8, seed)


@pytest.mark.parametrize("ng_of_tiles", [[1], [8], [3, 1], [1, 8, 2], [8, 8, 1, 5]])
def test_epilogue_hold_last_tile(ng_of_tiles):
    """The last tile of a CTA: no next tile, so nobody arrives on EMPTY of the held buffer and the stager has left."""
    for nch in (1, 2, 5):
        for seed in range(12):
            run(ng_of_tiles, nch, 8, seed)
