"""Model check of scan3.cu's ring hand-over: a tile of nch chunks takes nch stages, each ring buffer goes back to the
stagers as soon as its stage has been read, and a tile's last buffer goes back only after the tile's epilogue (for
k <= 32 it holds the parked sums meanwhile).  The stagers wait on EMPTY from stage 3 on, so they can fill all three
buffers ahead of the scanners, and after their last stage they take the arrivals of the last three stages.

One stager role and W scanner warps.  FULL(b) is an mbarrier per ring buffer (every scanner warp waits on the phase
parity it tracks in a bit mask, as the kernel does); EMPTY(b) is a named barrier that completes when ALL scanner warps
have arrived and the stager syncs; BAR_SCAN is a named barrier of the W scanner warps.  The tile descriptors sit in a
ring of four slots: the kernel's prologue writes tiles 0 and 1, and at stage 0 of tile n the stager publishes tile
n + 1 into slot (n + 1) % 4.  The tile list ends with an empty descriptor (ng = 0), which stops both roles.

Random interleavings check: no deadlock; the stager never rewrites a buffer some warp still reads or one that holds
sums still to be read; a warp reads a buffer only when it holds the warp's stage, and sums only of its own tile; a
FULL phase never completes twice before every warp consumed it (the parity bit would alias); the warps last read
stages at most three apart; a warp never arrives
twice on one EMPTY generation (the named barrier would complete without the stager); no descriptor slot is rewritten
while a warp still reads the tile it holds, and every descriptor is published before anyone reads it; every EMPTY
arrival is taken by the time both roles have left."""
import random

import pytest

SLOTS = 4


def ring_next(b):
    return 0 if b == 2 else b + 1


def stager(tiles, nch, st, W):
    b = gs = 0
    n = 0
    while tiles[n]:                                           # ng of slot n (written before the stager reads it)
        assert st["slot"][n % SLOTS] == n, f"stager reads slot {n % SLOTS} holding tile {st['slot'][n % SLOTS]}"
        for ch in range(nch):
            if gs >= 3:
                yield from sync_empty(st, b, W)
            if ch == 0 and n > 0:                             # publish tile n + 1 (claimed during tile n - 1)
                s = (n + 1) % SLOTS
                old = st["slot"][s]
                if old is not None:
                    assert all(t > old for t in st["tile_of"]), \
                        f"slot {s} (tile {old}) rewritten while warps are at tiles {st['tile_of']}"
                st["slot"][s] = n + 1
            assert st["readers"][b] == 0, f"buffer {b} rewritten while read (stage {gs})"
            assert st["holders"][b] == 0, f"buffer {b} rewritten while it holds sums still to be read (stage {gs})"
            assert all(c >= st["full_done"][b] for c in st["consumed"][b]), f"FULL({b}) phase would alias at stage {gs}"
            st["stage"][b] = gs
            st["sums"][b] = None
            st["full_done"][b] += 1
            yield "progress"
            b = ring_next(b)
            gs += 1
        n += 1
    for s in range(max(gs - 3, 0), gs):                       # the arrivals of the last three stages
        yield from sync_empty(st, s % 3, W)


def sync_empty(st, b, W):
    """bar.sync EMPTY(b) by the stager: completes when every scanner warp has arrived."""
    while st["empty_arrivals"][b] < W:
        yield "blocked"
    st["empty_arrivals"][b] -= W
    st["empty_pending"][b] = [False] * W


def arrive_empty(st, w, b):
    assert not st["empty_pending"][b][w], f"warp {w} arrived twice on one EMPTY({b}) generation"
    st["empty_pending"][b][w] = True
    st["empty_arrivals"][b] += 1


def scan_barrier(st, W):
    """bar.sync BAR_SCAN over the W scanner warps."""
    gen = st["bar_gen"]
    st["bar_count"] += 1
    if st["bar_count"] == W:
        st["bar_count"] = 0
        st["bar_gen"] += 1
    while st["bar_gen"] == gen:
        yield "blocked"


def read_descriptor(st, n):
    assert st["slot"][n % SLOTS] == n, f"tile {n}: slot {n % SLOTS} holds tile {st['slot'][n % SLOTS]}"


def scanner(w, tiles, nch, mode, st, W, rng):
    b = gs = 0
    ph = 0
    n = 0
    while True:
        st["tile_of"][w] = n
        read_descriptor(st, n)
        ng = tiles[n]
        if not ng:
            break
        bl = None
        for it in range(nch):
            while not st["full_done"][b] > st["consumed"][b][w]:    # mbarrier.try_wait.parity
                yield "blocked"
            assert (st["consumed"][b][w] & 1) == ((ph >> b) & 1), "parity mask out of step with the phases consumed"
            st["consumed"][b][w] += 1
            ph ^= 1 << b
            assert st["stage"][b] == gs, f"warp {w} stage {gs}: buffer {b} holds {st['stage'][b]}"
            st["pos"][w] = gs
            st["readers"][b] += 1
            yield "progress"
            assert st["stage"][b] == gs, f"warp {w} stage {gs}: buffer {b} rewritten while read"
            st["readers"][b] -= 1
            if it + 1 < nch:
                arrive_empty(st, w, b)
                yield "progress"
            else:
                bl = b
            b = ring_next(b)
            gs += 1
        last = gs - 1
        if mode == "cand":
            # k <= 32: the last buffer becomes the tile's sum area; warp w runs query w of the tile
            yield from scan_barrier(st, W)
            assert st["readers"][bl] == 0, "sums written while a warp still reads the last buffer"
            assert st["stage"][bl] == last, "last buffer rewritten before its sums were written"
            st["sums"][bl] = n
            st["holders"][bl] += 1
            yield "progress"
            yield from scan_barrier(st, W)
            if w < ng:
                for _ in range(rng.randint(1, 4)):                  # stats, bisection and append passes
                    assert st["sums"][bl] == n and st["stage"][bl] == last, f"warp {w} tile {n}: sums overwritten"
                    read_descriptor(st, n)
                    yield "progress"
            st["holders"][bl] -= 1
        else:
            # dense stores, or the k > 32 block epilogue: the descriptor is read throughout, the ring not at all; the
            # block epilogue's barriers are the same for every warp of the tile
            for _ in range(ng if mode == "list" else rng.randint(0, 3)):
                read_descriptor(st, n)
                if mode == "list":
                    yield from scan_barrier(st, W)
                yield "progress"
        read_descriptor(st, n)
        arrive_empty(st, w, bl)
        n += 1
        st["tile_of"][w] = n                                  # the warp reads tile n's descriptor no more
        yield "progress"
    st["pos"][w] = 1 << 30                                    # done: no longer bounds the drift


def run(ng_of_tiles, nch, W, mode, seed):
    rng = random.Random(seed)
    tiles = list(ng_of_tiles) + [0]                           # the descriptor after a CTA's last tile is empty
    st = {"stage": {0: None, 1: None, 2: None}, "readers": {0: 0, 1: 0, 2: 0}, "holders": {0: 0, 1: 0, 2: 0},
          "sums": {0: None, 1: None, 2: None}, "full_done": {0: 0, 1: 0, 2: 0},
          "consumed": {b: [0] * W for b in range(3)}, "empty_arrivals": {0: 0, 1: 0, 2: 0},
          "empty_pending": {b: [False] * W for b in range(3)}, "pos": [0] * W, "bar_count": 0, "bar_gen": 0,
          "slot": {0: 0, 1: 1, 2: None, 3: None}, "tile_of": [0] * W}
    roles = {"S": stager(tiles, nch, st, W)}
    roles.update({f"C{w}": scanner(w, tiles, nch, mode, st, W, rng) for w in range(W)})
    live = set(roles)
    blocked = set()                                           # roles that made no progress since the last progress
    drift = 0
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
        on = [p for p in st["pos"] if p < (1 << 30)]
        if on:
            drift = max(drift, max(on) - min(on))
    assert drift <= 3, f"scanner warps drifted {drift} stages apart"
    assert all(v == 0 for v in st["readers"].values())
    assert all(v == 0 for v in st["holders"].values())
    assert all(v == 0 for v in st["empty_arrivals"].values()), f"EMPTY arrivals left: {st['empty_arrivals']}"


NCH = [1, 2, 3, 12, 64]
MODES = ["cand", "dense", "list"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("nch", NCH)
@pytest.mark.parametrize("W", [1, 2, 8])
def test_ring_any_tile_length(nch, W, mode):
    for ntiles in (1, 2, 5):
        for seed in range(4 if nch < 64 else 2):
            run([W] * ntiles, nch, W, mode, seed)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("nch", NCH)
def test_ring_varying_ng(nch, mode):
    """Consecutive tiles of 1..8 queries, so some warps have no query and go straight on."""
    for seed in range(16 if nch < 64 else 4):
        rng = random.Random(1000 + seed)
        ng_of_tiles = [rng.randint(1, 8) for _ in range(rng.randint(1, 7))]
        run(ng_of_tiles, nch, 8, mode, seed)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ng_of_tiles", [[], [1], [8], [3, 1], [1, 8, 2], [8, 8, 1, 5]])
def test_ring_last_tile(ng_of_tiles, mode):
    """A CTA's last tile (and a CTA with no tile): the stager takes the arrivals of the last stages and leaves."""
    for nch in NCH:
        for seed in range(6 if nch < 64 else 2):
            run(ng_of_tiles, nch, 8, mode, seed)
