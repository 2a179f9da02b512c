"""GPU tier (-m gpu): seeded fuzzing of the range-proof verifiers that carry state from one call to the next or take a transcript per
proof, against the oracle's verdict of each proof alone.

1. bp.MixedVerifier on three reserved mixes: every (n, m) of the reference grid at small capacities (24 classes, the most a mix holds);
   one (64, 1) class of 200 slots (no conditional node, seven chunks); (64, 1) of 192 slots beside its alias (32, 2), (8, 4) and a
   (64, 64) class (k = 12).  Each round draws a live count per class from {0, 1, 31, 32, 33, capacity, random}, mutates a third of the
   items and verifies through begin, begin_each or verify_mixed on the service context.  Between rounds come calls that do not fit (an
   unreserved class, one proof over a capacity) and the fitting call after them, a profiled call (direct launches) and the clean call
   after it, a reserved BatchVerifier and an MSM on the same context.  Scripted rounds leave invalid proofs in every slot from the chunk
   that straddles the next round's live count on, reach the whole-class level of the reject path on a reserved class (and its partial
   last chunk alone), and make every class of the grid the only failing one.  Every call's verdicts equal verify_mixed(_each) on an
   unreserved context and the oracle's; a clean fitting call costs exactly the clean launch delta, a fitting call with a failing admitted
   proof more.
2. Reserving a mix again replaces it; a refused reserve keeps the previous one.
3. Records no transcript operation of the suite reaches: random sponges at every position 0..165, pos_begin 0, pos or random below it,
   random cur_flags, with proofs the oracle made under them; then the records changed in cur_flags only, in one sponge bit, in pos or in
   pos_begin, or made malformed.
4. Launch groups of 2 x 1024 and 5 x 40 under per-proof records, with proof and record mutations.

Seeds (random.Random): part 1 SEED + 100 * mix + round (mix 0 grid, 1 one class, 2 large and small), part 2 SEED + 1000, part 3 SEED +
2000 (the records) and SEED + 2001 (their mutations), part 4 SEED + 3000 + 100 * batches + round.  Every item records its mutation; a
mismatch names the test, seed, round, item, mutation, got and want."""
import random

import pytest

from oracle_binding import L_ORDER as l
from test_gpu_geometry import GRID, _cell
from test_gpu_group_check import LABEL, _expected
from test_gpu_large_aggregation import _cell as _large_cell
from test_gpu_mixed_service import Service, oracle, tx
from test_gpu_per_proof_transcripts import Pool, _contexts, _device_each, _prove, _want, malformed_record
from test_gpu_verifier_fuzz import (ALIASES, FORMAT_ERROR, INVALID_BITSIZE, INVALID_GENERATORS_LENGTH, KEEP_LENGTH, MIX_CELLS, OK, RESIZE,
                                    VERIFICATION_ERROR, _diff, _mutate_rp, _rp_admitted, _rp_category, mutate, rp_fields)

SEED = 20261018
REC = 203
ROUNDS = 10


def le(x, n=32):
    return x.to_bytes(n, "little")


def _plus_one(proof):
    """t_x + 1: well-formed, invalid"""
    return proof[:128] + le((int.from_bytes(proof[128:160], "little") + 1) % l) + proof[160:]


def _plen(n, m):
    return 32 * (9 + 2 * ((n * m).bit_length() - 1))


# ---------------------------------------------------------------------------------------------------------------------- the mixes
GRID_MIX = {c: 1 + i % 4 if c[0] * c[1] >= 512 else (1, 31, 32, 33, 2, 40)[i % 6] for i, c in enumerate(GRID)}
MIXES = [  # (name, mix, the table's parties, a proof of an admitted class outside the mix or None)
    ("grid", GRID_MIX, 32, None),
    ("one class", {(64, 1): 200}, 32, (8, 2)),
    ("large and small", {(64, 1): 192, (32, 2): 40, (8, 4): 33, (64, 64): 3}, 64, (16, 4)),
]
STALE = {"grid": ((8, 8), 20), "one class": ((64, 1), 70), "large and small": ((64, 1), 100)}    # class, live count after the stale round
NAMED = {0: "0", 1: "1", 31: "31", 32: "32", 33: "33"}


def _labels(v, cap):
    """what a live count v of a class of capacity cap stands for"""
    out = {NAMED[v]} if v in NAMED else set()
    if v == cap:
        out.add("capacity")
    return out or {"random"}


def _required(cap):
    unnamed = [v for v in range(cap + 1) if v not in NAMED and v != cap]
    return {NAMED[v] for v in NAMED if v <= cap} | {"capacity"} | ({"random"} if unnamed else set()), unnamed


def test_service_fuzz_mixes():
    """the grid mix holds every cell, capacities 1, 31, 32 and 33 among them and 1-4 where k >= 9; the stale classes have a live count
    that is not a multiple of RP_CHUNK = 32 below their capacity; the large mix has a class with k >= 12 and the alias of (64, 1)"""
    assert set(GRID_MIX) == set(GRID) and len(GRID_MIX) == 24 and {1, 31, 32, 33} <= set(GRID_MIX.values())
    assert all(1 <= c <= 4 for (n, m), c in GRID_MIX.items() if n * m >= 512)
    for name, mix, _, _ in MIXES:
        c, live = STALE[name]
        assert live % 32 and live < mix[c] and mix[c] > 32 * (live // 32) + 1, name
    large = MIXES[2][1]
    assert any(n * m >= 1 << 12 for n, m in large) and ((64, 1), (32, 2)) in ALIASES and large[(64, 1)] >= 161


class _Service(Service):
    """test_gpu_mixed_service's Service on a table of 64 generators and `parties` parties (a k >= 12 class needs more than 32)"""

    def __init__(self, mix, parties=32):
        import bulletproofs_b200 as bp
        self.ctx = bp.Context(0)
        self.gens = bp.Gens(self.ctx, 64, parties)
        self.v = bp.MixedVerifier(self.ctx, self.gens, mix)
        self.clean = None


# ---------------------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


@pytest.fixture(scope="module")
def og64(orc):
    return orc.gens(64, 64)


@pytest.fixture(scope="module")
def ref(built):
    """a context that never reserves anything, with a (64, 32) and a (64, 64) table: the direct launches of every mixed call"""
    import bulletproofs_b200 as bp
    ctx = bp.Context(0)
    tables = {32: bp.Gens(ctx, 64, 32), 64: bp.Gens(ctx, 64, 64)}
    yield ctx, tables
    for g in tables.values():
        g.close()
    ctx.close()


@pytest.fixture(scope="module")
def cells(orc, og, og64):
    """{(n, m): [(proof, commitments)]}: the distinct oracle proofs of every grid cell (fresh LABEL transcript) and of (64, 64)"""
    out = {}
    for n, m in GRID:
        proofs, Vs, plen = _cell(orc, og, n, m)
        out[(n, m)] = [(proofs[i * plen:(i + 1) * plen], Vs[32 * m * i:32 * m * (i + 1)]) for i in range(4)]
    _, _, _, proofs, Vs = _large_cell(None, orc, None, (None, og64), 64, 64)
    plen = _plen(64, 64)
    out[(64, 64)] = [(proofs[i * plen:(i + 1) * plen], Vs[2048 * i:2048 * (i + 1)]) for i in range(len(proofs) // plen)]
    return out


@pytest.fixture(scope="module")
def pool64(orc, og):
    return Pool(orc, og, 64, 1, 4, 500)


def _arbitrary_records():
    """166 records: a random 200-byte sponge, pos 0..165, pos_begin 0, pos or random up to pos in turn, random cur_flags"""
    rnd = random.Random(SEED + 2000)
    return [rnd.randbytes(200) + bytes([pos, (0, pos, rnd.randint(0, pos))[pos % 3], rnd.randrange(256)]) for pos in range(166)]


@pytest.fixture(scope="module")
def arb(orc, og):
    """[(n, m, record, proof, commitments)]: one (64, 1) oracle proof under each of the 166 records of _arbitrary_records, and (8, 2) and
    (16, 4) proofs under eight of them"""
    recs = _arbitrary_records()
    out = []
    for i, r in enumerate(recs):
        proofs, Vs = _prove(orc, og, r, 64, 1, 1, 40000 + i)
        out.append((64, 1, r, proofs, Vs))
    for n, m in ((8, 2), (16, 4)):
        for i in (0, 1, 2, 83, 120, 163, 164, 165):
            proofs, Vs = _prove(orc, og, recs[i], n, m, 1, 50000 + 1000 * n + i)
            out.append((n, m, recs[i], proofs, Vs))
    return out


def test_arbitrary_records_reach_every_position():
    """the records of part 3 hold every pos, the three pos_begin forms and more than a hundred distinct cur_flags"""
    recs = _arbitrary_records()
    assert [r[200] for r in recs] == list(range(166)) and all(r[201] <= r[200] for r in recs)
    assert sum(r[201] == 0 < r[200] for r in recs) > 50 and sum(r[201] == r[200] > 0 for r in recs) > 50
    assert sum(0 < r[201] < r[200] for r in recs) > 20 and len({r[202] for r in recs}) > 100


# ---------------------------------------------------------------------------------------------------------------------- part 1 helpers
def _mutate_item(rnd, it, pool, by_len, by_m, resize=True):
    """_mutate_rp on [proof, commitments, n, name] (in place); a geometry without an alias of its length gets a field mutation instead"""
    n, m = it[2], len(it[1]) // 32
    if any(b[0] * b[1] == n * m for _, b in ALIASES):
        _mutate_rp(rnd, it, pool, by_len, by_m, resize)
    else:
        it[0], it[3] = mutate(rnd, it[0], rp_fields(len(it[0])), by_len[len(it[0])], KEEP_LENGTH + (RESIZE if resize else ()))


def _interleave(rnd, per, extras=()):
    """the items of every class merged in a random order that keeps each class's own order (its slot order); extras anywhere"""
    lists = [list(v) for v in per.values()] + [[e] for e in extras]
    tags = [i for i, lst in enumerate(lists) for _ in lst]
    rnd.shuffle(tags)
    its = [iter(lst) for lst in lists]
    return [next(its[t]) for t in tags]


def _check_call(bp, orc, og, s, ref_ctx, ref_gens, items, mode, seed_bytes, tag, seed, round_):
    """one call on the service context: items [proof, commitments, n, name, record]; mode begin (one LABEL transcript), begin_each (the
    records) or verify_mixed (blocking, LABEL).  Asserts verdicts == verify_mixed(_each) on the unreserved context == the oracle's;
    returns (verdicts, launch delta)"""
    triples = [tuple(it[:3]) for it in items]
    each = mode == "begin_each"
    l0 = s.ctx.launches
    if mode == "begin":
        s.v.begin(bp.Transcript(LABEL), triples, seed=seed_bytes)
        got = s.v.finish()
    elif each:
        s.v.begin_each([(bp.Transcript(state=it[4]), *t) for it, t in zip(items, triples)], seed=seed_bytes)
        got = s.v.finish()
    else:
        got = bp.verify_mixed(s.ctx, s.gens, bp.Transcript(LABEL), triples, seed=seed_bytes)
    dl = s.ctx.launches - l0
    if each:
        direct = bp.verify_mixed_each(ref_ctx, ref_gens, [(bp.Transcript(state=it[4]), *t) for it, t in zip(items, triples)], seed=seed_bytes)
    else:
        direct = bp.verify_mixed(ref_ctx, ref_gens, bp.Transcript(LABEL), triples, seed=seed_bytes)
    want = oracle(orc, og, triples, [it[4] for it in items] if each else None)
    names = [it[3] for it in items]
    assert got == want, _diff(f"{tag} {mode}", seed, round_, names, got, want)
    assert direct == want, _diff(f"{tag} {mode} (unreserved context)", seed, round_, names, direct, want)
    return got, dl


class _MixFuzz:
    """one reserved mix under fuzz: its service context, the unreserved reference, the item sources and what the calls reached"""

    def __init__(self, bp, orc, name, mix, parties, og, ref, cells, recs):
        self.bp, self.orc, self.name, self.mix, self.parties, self.og = bp, orc, name, mix, parties, og
        self.ref_ctx, self.ref_gens = ref[0], ref[1][parties]
        self.cells = cells
        self.pool = {c: cells[c] for c in MIX_CELLS}
        self.by_len, self.by_m = {}, {}
        for (n, m), src in cells.items():
            if m <= parties:
                self.by_len.setdefault(len(src[0][0]), []).extend(p for p, _ in src)
                self.by_m.setdefault(m, []).extend(V for _, V in src)
        self.recs = recs                                    # [(record, proof, commitments)] of (64, 1) under records of their own
        self.lab = orc.transcript(LABEL)[:REC]
        self.others = sorted({r for r, _, _ in recs} | set(_contexts(orc)))
        self.proof_bytes = sum(c * _plen(n, m) for (n, m), c in mix.items())
        self.commit_bytes = sum(32 * c * m for (n, m), c in mix.items())
        self.s = _Service(mix, parties)
        # coverage
        self.live_seen = {c: set() for c in mix}
        self.calls = []                                     # (shared | records, fits) of every call in order
        self.codes, self.alone, self.whole, self.last_chunk, self.whole_beside_passing = set(), set(), set(), set(), False
        self.stale_checked = self.prof_checked = False

    def close(self):
        self.s.close()

    # ---- items
    def valid(self, rnd, c, count, each):
        """count valid items of class c; under records, half of the (64, 1) ones are proofs made under records of their own"""
        src = self.cells[c]
        j0 = rnd.randrange(len(src))
        out = [[*src[(j0 + i) % len(src)], c[0], "valid", self.lab] for i in range(count)]
        if each and c == (64, 1):
            for it in out:
                if rnd.random() < 0.5:
                    r, p, V = rnd.choice(self.recs)
                    it[:] = [p, V, 64, "valid under its own record", r]
        return out

    def admitted(self, it):
        return _rp_admitted(len(it[0]), it[2], len(it[1]) // 32, gens_parties=self.parties)

    def mutate(self, rnd, per, each, classes=None):
        """a third of the items of `classes` (default: all) get one mutation, a record mutation for a third of them under records; an
        item that leaves its class (a resized proof) is followed by a valid one, so the class keeps its live count"""
        pool = [(c, it) for c, its in per.items() if classes is None or c in classes for it in its]
        for c, it in rnd.sample(pool, len(pool) // 3):
            if each and rnd.random() < 0.33:
                kind = rnd.randrange(4)
                if kind == 0:
                    it[4], it[3] = malformed_record(rnd, rnd.randrange(2)), "malformed record"
                elif kind == 1:
                    r = bytearray(it[4]); r[202] ^= rnd.randrange(1, 256); it[4], it[3] = bytes(r), f"record's cur_flags = {r[202]}"
                elif kind == 2:
                    it[4], it[3] = rnd.choice([r for r in self.others if r != it[4]]), "another proof's record"
                else:
                    o = rnd.choice(pool)[1]
                    if o is not it and o[4] != it[4]:
                        it[4], o[4] = o[4], it[4]; it[3], o[3] = "records swapped", "records swapped"
                continue
            sub = it[:4]
            _mutate_item(rnd, sub, self.pool, self.by_len, self.by_m)
            it[:4] = sub
            if self.admitted(it) != c:
                per[c] += self.valid(rnd, c, 1, each)

    def extras(self):
        """proofs the parameters reject: n = 12 (InvalidBitsize), m above the table's parties (InvalidGeneratorsLength), m = 3"""
        (p82, V82), (p84, V84) = self.cells[(8, 2)][0], self.cells[(8, 4)][1]
        over = self.parties + 8
        return [[p82, V82, 12, "n = 12", self.lab], [p82, V82 * (over // 2), 8, f"m = {over} above the table's parties", self.lab],
                [p84, V84[:96], 8, "m = 3", self.lab]]

    def trim(self, rnd, items):
        """drop proofs the parameters reject until the buffers are no larger than those of the mix at capacity, so the call fits"""
        while self.fits(items, self.classes(items, None)) is None:
            items.remove(rnd.choice([it for it in items if self.admitted(it) is None]))
        return items

    # ---- one call
    def classes(self, items, want):
        """{class: categories of its admitted items in slot order} (categories only when the verdicts are given)"""
        out = {}
        for j, it in enumerate(items):
            c = self.admitted(it)
            if c is not None:
                out.setdefault(c, []).append(None if want is None else _rp_category(self.orc, want[j], it[0], it[1]))
        return out

    def fits(self, items, classes):
        """True when the call fits the mix as bpmsm.h defines it, False when a class is not reserved or over its capacity, None when only
        the buffer sizes exceed the mix's (the engine may take either path)"""
        if any(c not in self.mix or len(v) > self.mix[c] for c, v in classes.items()):
            return False
        if sum(len(it[0]) for it in items) > self.proof_bytes or sum(32 * (len(it[1]) // 32) for it in items) > self.commit_bytes:
            return None
        return True

    def call(self, rnd, items, tag, seed, round_, mode=None, direct=False):
        """items on the service in a random mode (or `mode`); checks the verdicts and the launch delta: a fitting call that admits nothing
        launches nothing, a clean one costs the clean delta, one with a failing admitted proof more; a call on the direct launches (not
        fitting, or `direct`: profiled) never costs the clean delta when it is clean.  Returns (verdicts, classes, fits)"""
        mode = mode or rnd.choice(("begin", "begin_each", "verify_mixed"))
        want, dl = _check_call(self.bp, self.orc, self.og, self.s, self.ref_ctx, self.ref_gens, items, mode, rnd.randbytes(32),
                               f"test_reserved_mix_fuzz[{self.name}] {tag}", seed, round_)
        classes = self.classes(items, want)
        fit = self.fits(items, classes)
        wrong = {c for c, cats in classes.items() if "wrong" in cats}
        where = f"test_reserved_mix_fuzz[{self.name}] {tag} seed {seed} round {round_} {mode}: launches {dl}, clean {self.s.clean}, failing {wrong}"
        if fit and not direct:
            if not classes:
                assert dl == 0, where
            elif not wrong:
                assert dl == self.s.clean, where
            else:
                assert dl > self.s.clean, where
        elif fit is not None and classes and not wrong:
            assert dl != self.s.clean, where
        self.calls.append(("records" if mode == "begin_each" else "shared", fit and not direct))
        self.codes |= set(want)
        if fit and not direct:
            for c, cap in self.mix.items():
                self.live_seen[c] |= _labels(len(classes.get(c, [])), cap)
            if len(wrong) == 1:
                self.alone |= wrong
            for c, cats in classes.items():
                chunks = [i // 32 for i, x in enumerate(cats) if x == "wrong"]
                if len(cats) >= 161 and len(cats) % 32:
                    if len(set(chunks)) > 4:
                        self.whole.add(c)
                        self.whole_beside_passing |= any(d not in wrong for d in classes if d != c)
                    if set(chunks) == {len(cats) // 32}:
                        self.last_chunk.add(c)
        return want, classes, fit

    # ---- between rounds
    def clean_call(self, rnd, tag, seed, round_, direct=False):
        """valid proofs, up to five per class, in a few classes: fits"""
        live = {c: rnd.randint(0, min(cap, 5)) if rnd.random() < 0.6 else 0 for c, cap in self.mix.items()}
        c0 = rnd.choice(list(self.mix))
        live[c0] = max(1, live[c0])
        mode = rnd.choice(("begin", "begin_each", "verify_mixed"))
        items = _interleave(rnd, {c: self.valid(rnd, c, k, mode == "begin_each") for c, k in live.items()})
        _, _, fit = self.call(rnd, items, tag, seed, round_, mode, direct)
        assert fit is True

    def batch_verifier(self, rnd, seed, round_):
        """a reserved BatchVerifier of 2 x 16 (64, 1) proofs on the service context, one of them t_x + 1"""
        bp = self.bp
        src = self.cells[(64, 1)]
        items = [src[i % len(src)] for i in range(32)]
        bad = rnd.randrange(32)
        items[bad] = (_plus_one(items[bad][0]), items[bad][1])
        bv = bp.BatchVerifier(self.s.ctx, self.s.gens, bp.Transcript(LABEL), 64, 1, 16, 2)
        bv.begin(b"".join(p for p, _ in items), b"".join(V for _, V in items), rnd.randbytes(32))
        got = list(bv.finish())
        want = oracle(self.orc, self.og, [(p, V, 64) for p, V in items])
        assert got == want and bv.batch_ok == [int(bad >= 16), int(bad < 16)], (f"BatchVerifier seed {seed} round {round_}", got, bv.batch_ok)

    def msm(self, rnd, seed, round_):
        pts = b"".join(p[:32] for c in sorted(self.cells) for p, _ in self.cells[c])
        scalars = b"".join(le(rnd.randrange(l)) for _ in range(len(pts) // 32))
        assert self.s.ctx.msm(scalars, pts) == self.orc.msm(scalars, pts), f"MSM seed {seed} round {round_}"


def _live_schedule(rnd, mix, fixed):
    """{round: {class: live count}}: fixed[(round, class)] where given; elsewhere every live-count form a class admits at least once, then
    random forms"""
    sched = {r: {} for r in range(ROUNDS)}
    for c, cap in mix.items():
        need, unnamed = _required(cap)
        free = []
        for r in range(ROUNDS):
            if (r, c) in fixed:
                sched[r][c] = fixed[(r, c)]
                need -= _labels(fixed[(r, c)], cap)
            else:
                free.append(r)
        rnd.shuffle(free)
        need = sorted(need)
        assert len(need) <= len(free), (c, need)
        value = {"capacity": cap, **{v: k for k, v in NAMED.items()}}
        for i, r in enumerate(free):
            form = need[i] if i < len(need) else rnd.choice(sorted(_required(cap)[0]))
            sched[r][c] = rnd.choice(unnamed) if form == "random" else value[form]
    return sched


# ---------------------------------------------------------------------------------------------------------------------- 1. reserved mixes
@pytest.mark.gpu
@pytest.mark.parametrize("which", range(len(MIXES)), ids=[m[0].replace(" ", "_") for m in MIXES])
def test_reserved_mix_fuzz(orc, og, og64, ref, cells, pool64, arb, which):
    """ROUNDS rounds on one reserved mix, the scripted ones at fixed rounds: 2 fills the stale class to capacity with t_x + 1 from the
    chunk that straddles round 3's live count on, 3 is clean with that live count and must cost the clean delta; with a (64, 1) class of
    161 or more slots, 5 puts wrong proofs in five or more of its chunks (the last, partial one included) and 7 only in its partial last
    chunk, every other class passing.  After rounds 6 and 8 the round's items plus a proof that does not fit, then a clean fitting call;
    after round 4 a profiled call, then a clean one; a reserved BatchVerifier after rounds 3 and 8, an MSM after round 5; in the grid
    mix, three calls after each of rounds 0-7 in each of which one class alone fails."""
    import bulletproofs_b200 as bp
    name, mix, parties, outside = MIXES[which]
    recs = list(pool64.entries) + [(r, p, V) for n, m, r, p, V in arb if n == 64]
    F = _MixFuzz(bp, orc, name, mix, parties, og64 if parties == 64 else og, ref, cells, recs)
    rnd0 = random.Random(SEED + 100 * which)
    big = (64, 1) if mix.get((64, 1), 0) >= 161 else None
    stale_c, stale_live = STALE[name]
    fixed = {(2, stale_c): mix[stale_c], (3, stale_c): stale_live}
    if big:
        cap = mix[big]
        whole_live = rnd0.choice([v for v in range(161, cap + 1) if v % 32])
        last_live = rnd0.choice([v for v in range(161, cap + 1) if v % 32 and v != whole_live])
        fixed.update({(5, big): whole_live, (7, big): last_live})
    sched = _live_schedule(rnd0, mix, fixed)
    modes = ["begin", "begin_each", "verify_mixed"] + [rnd0.choice(("begin", "begin_each", "verify_mixed")) for _ in range(ROUNDS - 3)]
    solo = sorted(mix) if name == "grid" else []
    try:
        F.s.clean = _check_call(bp, orc, F.og, F.s, F.ref_ctx, F.ref_gens, F.valid(rnd0, stale_c, 1, False), "begin", bytes(32),
                                f"test_reserved_mix_fuzz[{name}] clean delta", SEED + 100 * which, "-")[1]
        for round_ in range(ROUNDS):
            seed = SEED + 100 * which + round_
            rnd = random.Random(seed)
            each = modes[round_] == "begin_each"
            per = {c: F.valid(rnd, c, k, each) for c, k in sched[round_].items()}
            extras = []
            if round_ == 2:                              # the stale class at capacity, t_x + 1 from the straddling chunk on
                start = 32 * (stale_live // 32)
                for it in per[stale_c][start:]:
                    it[0], it[3], it[4] = _plus_one(it[0]), "t_x + 1 (stale next round)", F.lab
                F.mutate(rnd, per, each, [c for c in per if c != stale_c])
            elif round_ == 5 and big:                    # wrong proofs in five or more chunks of the big class, the last one included
                nch = -(-whole_live // 32)
                bad = {32 * ch + rnd.randrange(min(32, whole_live - 32 * ch)) for ch in rnd.sample(range(nch - 1), rnd.randint(4, nch - 1)) + [nch - 1]}
                for i in bad:
                    per[big][i][0], per[big][i][3] = _plus_one(per[big][i][0]), "t_x + 1"
                for i in rnd.sample([i for i in range(whole_live) if i not in bad], whole_live // 3):
                    sub = per[big][i][:4]; _mutate_item(rnd, sub, F.pool, F.by_len, F.by_m, resize=False); per[big][i][:4] = sub
            elif round_ == 7 and big:                    # the only wrong proof in the partial last chunk of the big class
                it = per[big][rnd.randrange(32 * (last_live // 32), last_live)]
                it[0], it[3] = _plus_one(it[0]), "t_x + 1 in the partial last chunk"
            elif round_ != 3:
                F.mutate(rnd, per, each)
                if round_ % 2:
                    extras = F.extras()
            items = F.trim(rnd, _interleave(rnd, per, extras)) or F.extras()          # no live proof: a call the parameters decide
            want, classes, fit = F.call(rnd, items, "round", seed, round_, modes[round_])
            assert fit is True and all(len(classes.get(c, [])) == k for c, k in sched[round_].items()), (seed, round_, fit)
            if round_ == 3:
                assert all(w == OK for w in want)
                F.stale_checked = True
            if round_ in (6, 8):                         # the round's items and one proof that does not fit; then a fitting call
                if outside:
                    p, V = rnd.choice(cells[outside])
                    more = [[p, V, outside[0], f"an unreserved {outside} proof", F.lab]]
                else:
                    c = min(mix, key=lambda d: mix[d] - len(classes.get(d, [])))
                    more = F.valid(rnd, c, mix[c] - len(classes.get(c, [])) + 1, False)
                    for it in more:
                        it[3] = f"{c} over its capacity {mix[c]}"
                _, _, fit = F.call(rnd, items + F.extras() + more, "not fitting", seed, f"{round_} (not fitting)")
                assert fit is False
                F.clean_call(rnd, "after a call that did not fit", seed, f"{round_} (after not fitting)")
            if round_ == 4:                              # profiled: the direct launches; then the graph again
                F.s.ctx.prof_enable(True)
                try:
                    F.clean_call(rnd, "profiled", seed, f"{round_} (profiled)", direct=True)
                finally:
                    F.s.ctx.prof_enable(False)
                F.clean_call(rnd, "after profiling", seed, f"{round_} (after profiling)")
                F.prof_checked = True
            if round_ in (3, 8):
                F.batch_verifier(rnd, seed, round_)
            if round_ == 5:
                F.msm(rnd, seed, round_)
            for c in solo[3 * round_:3 * round_ + 3]:    # class c the only one failing
                live = {d: rnd.randint(0, min(cap, 3)) for d, cap in mix.items()}
                live[c] = max(1, live[c])
                each = rnd.random() < 0.5
                per = {d: F.valid(rnd, d, k, each) for d, k in live.items()}
                it = rnd.choice(per[c])
                it[0], it[3] = _plus_one(it[0]), "t_x + 1 (the only failing class)"
                _, classes, fit = F.call(rnd, _interleave(rnd, per), f"{c} alone failing", seed, f"{round_} ({c} alone)",
                                         "begin_each" if each else rnd.choice(("begin", "verify_mixed")))
                assert fit is True and {d for d, cats in classes.items() if "wrong" in cats} == {c}
    finally:
        F.close()
    # coverage: what each of the listed cases needs was reached
    missing = {c: sorted(_required(cap)[0] - F.live_seen[c]) for c, cap in mix.items() if _required(cap)[0] - F.live_seen[c]}
    assert not missing, f"live-count forms never run on a fitting call: {missing}"
    assert F.stale_checked, "no clean round after the stale class was filled with invalid proofs"
    if big:
        assert big in F.whole, "the whole-class level of the reject path was never reached on a reserved class"
        assert big in F.last_chunk, "no round had its only wrong proof in the partial last chunk of a class of 161 or more"
        if len(mix) > 1:
            assert F.whole_beside_passing, "no whole-class round beside passing classes"
    seq = [kind for kind, fits in F.calls]
    assert ("shared", "records") in zip(seq, seq[1:]), "shared transcript then records never in consecutive calls"
    assert ("records", "shared") in zip(seq, seq[1:]), "records then shared transcript never in consecutive calls"
    assert any(a[1] is False and b[1] is True for a, b in zip(F.calls, F.calls[1:])), "no call that did not fit followed by one that did"
    assert F.prof_checked
    assert F.codes >= {OK, VERIFICATION_ERROR, FORMAT_ERROR, INVALID_BITSIZE, INVALID_GENERATORS_LENGTH}, F.codes
    if solo:
        assert F.alone == set(mix), f"classes never the only failing one: {sorted(set(mix) - F.alone)}"


# ---------------------------------------------------------------------------------------------------------------------- 2. re-reserving
def _reserve(bp, ctx, gens, classes):
    """bp_rangeproof_verify_mixed_reserve over [(n, m, capacity)] exactly as given (a dict could not hold a duplicate class)"""
    arr = bp._c.c_uint32 * max(len(classes), 1)
    ctx._check(bp.lib().bp_rangeproof_verify_mixed_reserve(ctx._h, gens._h, len(classes), arr(*[c[0] for c in classes]),
                                                           arr(*[c[1] for c in classes]), arr(*[c[2] for c in classes])))


@pytest.mark.gpu
def test_reserving_again_replaces_the_mix_and_a_refused_reserve_keeps_it(orc, og64, ref, cells):
    """mix A, a round on it; then mix B with other classes on the same context: a call that fits only A takes the direct launches with A's
    verdicts, a call that fits B replays at B's clean delta (that of a fresh context with B).  Reserves refused for 25 classes, a duplicate
    class, zero capacity and m above the table's parties raise ERR_INVALID_ARGUMENT and leave B reserved"""
    import bulletproofs_b200 as bp
    A, B = {(64, 1): 40, (8, 2): 33}, {(16, 4): 33, (32, 2): 20, (8, 8): 5}
    seed = SEED + 1000
    rnd = random.Random(seed)
    ref_ctx, ref_gens = ref[0], ref[1][64]
    lab = orc.transcript(LABEL)[:REC]

    def items(counts, bad=0):
        out = [[*cells[c][i % len(cells[c])], c[0], "valid", lab] for c, k in counts.items() for i in range(k)]
        for it in rnd.sample(out, bad):
            it[0], it[3] = _plus_one(it[0]), "t_x + 1"
        rnd.shuffle(out)
        return out

    def run(s, its, tag):
        return _check_call(bp, orc, og64, s, ref_ctx, ref_gens, its, rnd.choice(("begin", "verify_mixed")), rnd.randbytes(32),
                           f"test_reserving_again {tag}", seed, "-")[1]

    fresh, s = _Service(B, parties=64), _Service(A, parties=64)
    try:
        clean_b = run(fresh, items({(16, 4): 3, (8, 8): 1}), "fresh B")
        clean_a = run(s, items({(64, 1): 40, (8, 2): 7}), "A")
        assert clean_a != clean_b and run(s, items({(64, 1): 33, (8, 2): 33}, bad=2), "A failing") > clean_a
        assert run(s, items({(64, 1): 1}), "A clean") == clean_a
        s.v = bp.MixedVerifier(s.ctx, s.gens, B)
        only_a = items({(64, 1): 30, (8, 2): 10})
        assert run(s, only_a, "only A after B") not in (clean_a, clean_b)
        assert run(s, items({(16, 4): 33, (32, 2): 20, (8, 8): 5}), "B full") == clean_b
        assert run(s, items({(32, 2): 12, (8, 8): 2}, bad=1), "B failing") > clean_b
        refused = [("25 classes", [(n, m, 1) for n, m in GRID] + [(64, 64, 1)], "1 to 24 classes"),
                   ("a duplicate class", [(16, 4, 3), (8, 2, 3), (16, 4, 5)], "duplicate"),
                   ("zero capacity", [(8, 2, 4), (16, 4, 0)], "zero capacity"),
                   ("m above the table's parties", [(8, 2, 4), (8, 128, 1)], "not admitted by the generators")]
        for what, classes, why in refused:
            with pytest.raises(bp.BpError) as e:
                _reserve(bp, s.ctx, s.gens, classes)
            assert e.value.code == bp.ERR_INVALID_ARGUMENT and why in str(e.value), (what, str(e.value))
            assert run(s, items({(16, 4): rnd.randint(1, 33), (32, 2): rnd.randint(0, 20)}), f"B after {what}") == clean_b, what
            assert run(s, only_a, f"only A after {what}") not in (clean_a, clean_b), what
        with pytest.raises(bp.BpError) as e:
            bp.MixedVerifier(s.ctx, s.gens, {(8, 2): 0})
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
        assert run(s, items({(8, 8): 5}), "B after a refused MixedVerifier") == clean_b
    finally:
        fresh.close()
        s.close()


# ---------------------------------------------------------------------------------------------------------------------- 3. arbitrary records
def _every_entry_point(bp, orc, og, ref, entries, want, tag, seed):
    """entries [(n, m, record, proof, commitments)], want the oracle's verdicts: verify_group_each on the direct and the graph path and
    verify_group_device_each with the records at byte 3 of a device buffer, over the (64, 1) entries as two batches (flags and device
    verdicts by the launch-group rule); verify_mixed_each over all on the unreserved context; MixedVerifier.begin_each over all on a
    reserved mix, at the clean delta when nothing fails inside the combination"""
    names = [f"({n},{m}) pos {r[200]} pos_begin {r[201]} cur_flags {r[202]}" for n, m, r, _, _ in entries]
    sd = random.Random(seed).randbytes(32)
    g = [(r, p, V) for (n, m, r, p, V) in entries if n == 64]
    gw = [w for e, w in zip(entries, want) if e[0] == 64]
    gnames = [x for e, x in zip(entries, names) if e[0] == 64]
    count, nb = len(g) // 2, 2
    g, gw, gnames = g[:count * nb], gw[:count * nb], gnames[:count * nb]
    failing = {b for b in range(nb) if any(_rp_category(orc, gw[i], g[i][1], g[i][2]) == "wrong" for i in range(b * count, (b + 1) * count))}
    ok_want, dev_want = _expected(gw, count, nb, failing)
    recs, proofs, Vs = b"".join(t for t, _, _ in g), b"".join(p for _, p, _ in g), b"".join(V for _, _, V in g)
    for path in ("direct", "graph"):
        ctx = bp.Context(0)
        gens = bp.Gens(ctx, 64, 32)
        try:
            if path == "graph":
                ctx._check(bp.lib().bp_rangeproof_verify_reserve(ctx._h, gens._h, 64, 1, count, nb))
            got, ok = bp.verify_group_each(ctx, gens, recs, proofs, Vs, 64, 1, count, nb, seed=sd)
            assert got == gw, _diff(f"{tag} verify_group_each {path}", seed, 0, gnames, got, gw)
            assert ok == ok_want, (tag, path, ok, ok_want)
            dgot, dok = _device_each(bp, ctx, gens, 64, 1, count, nb, g, sd, front=3)
            assert dgot == dev_want, _diff(f"{tag} verify_group_device_each {path}", seed, 0, gnames, dgot, dev_want)
            assert dok == ok_want, (tag, path, dok, ok_want)
        finally:
            gens.close(); ctx.close()
    each = [(bp.Transcript(state=r), p, V, n) for n, m, r, p, V in entries]
    got = bp.verify_mixed_each(ref[0], ref[1][32], each, seed=sd)
    assert got == want, _diff(f"{tag} verify_mixed_each", seed, 0, names, got, want)
    s = Service({(64, 1): 170, (8, 2): 8, (16, 4): 8})
    try:
        _, s.clean = s.run(tx(orc, og, {1: 3}), sd)
        got, dl = s.run(each, sd, each=True)
        assert got == want, _diff(f"{tag} MixedVerifier.begin_each", seed, 0, names, got, want)
        wrong = any(_rp_category(orc, w, p, V) == "wrong" for (n, m, r, p, V), w in zip(entries, want))
        assert dl > s.clean if wrong else dl == s.clean, (tag, dl, s.clean)
    finally:
        s.close()


@pytest.mark.gpu
def test_arbitrary_records_are_accepted_everywhere(orc, og, ref, arb):
    """the oracle's proofs under records with random sponges at every position: every entry point accepts all of them"""
    import bulletproofs_b200 as bp
    want = [_want(orc, og, n, m, [(r, p, V)])[0] for n, m, r, p, V in arb]
    assert want == [OK] * len(arb)
    entries = list(arb)
    random.Random(SEED + 2000).shuffle(entries)
    _every_entry_point(bp, orc, og, ref, entries, want, "test_arbitrary_records_are_accepted_everywhere", SEED + 2000)


@pytest.mark.gpu
def test_arbitrary_record_mutations(orc, og, ref, arb):
    """every record changed one way, in turn: cur_flags only (still accepted, by the oracle too), one sponge bit, pos moved, pos_begin
    moved (pos_begin <= pos < 166 kept), malformed (FormatError); every entry point gives the oracle's verdict for the changed record"""
    import bulletproofs_b200 as bp
    seed = SEED + 2001
    rnd = random.Random(seed)
    entries, kinds = [], {}
    for i, (n, m, r, p, V) in enumerate(arb):
        rec, pos, begin = bytearray(r), r[200], r[201]
        kind = ("cur_flags", "sponge bit", "pos", "pos_begin", "malformed")[i % 5]
        if kind == "pos" and begin == pos == 165 or kind == "pos_begin" and pos == 0:
            kind = "sponge bit"
        if kind == "cur_flags":
            rec[202] ^= rnd.randrange(1, 256)
        elif kind == "sponge bit":
            rec[rnd.randrange(200)] ^= 1 << rnd.randrange(8)
        elif kind == "pos":
            rec[200] = rnd.choice([q for q in range(begin, 166) if q != pos])
        elif kind == "pos_begin":
            rec[201] = rnd.choice([q for q in range(pos + 1) if q != begin])
        else:
            rec = bytearray(malformed_record(rnd, i % 2))
        entries.append((n, m, bytes(rec), p, V))
        kinds[i] = kind
    want = [_want(orc, og, n, m, [(r, p, V)])[0] for n, m, r, p, V in entries]
    for i, w in enumerate(want):
        if kinds[i] == "cur_flags":
            assert w == OK, f"the oracle rejects a proof whose record differs in cur_flags only: entry {i}"
        if kinds[i] == "malformed":
            assert w == FORMAT_ERROR
    assert set(kinds.values()) == {"cur_flags", "sponge bit", "pos", "pos_begin", "malformed"} and set(want) == {OK, VERIFICATION_ERROR, FORMAT_ERROR}
    _every_entry_point(bp, orc, og, ref, entries, want, "test_arbitrary_record_mutations", seed)


# ---------------------------------------------------------------------------------------------------------------------- 4. launch groups
GROUPS = [(2, 1024), (5, 40)]               # (batches, proofs per batch) of (64, 1)
LEVELS = ("none", "one", "few", "many")
RECORD_MUTATIONS = ("records swapped", "another proof's record", "malformed record", "cur_flags changed")


@pytest.mark.gpu
@pytest.mark.parametrize("nb,count", GROUPS)
def test_launch_group_fuzz_with_records(orc, og, pool64, arb, cells, nb, count):
    """launch groups of (64, 1) proofs under per-proof records (the pool's contexts and the random records), batches with 0, 1, 2-4 and more
    than 4 mutated proofs: proof mutations of the launch-group fuzz and record mutations (two records swapped, another proof's record, a
    malformed record, cur_flags changed).  verify_group_each on the direct and the graph path gives the oracle's verdicts and the per-batch
    flags; verify_group_device_each gives the flags and VerificationError for every proof without a code of its own in a failing batch
    (a malformed record is a rejected proof outside the combination)"""
    import bulletproofs_b200 as bp
    base = [(r, p, V) for r, p, V in pool64.entries] + [(r, p, V) for n, m, r, p, V in arb if n == 64]
    pool = {c: cells[c] for c in MIX_CELLS}
    by_len, by_m = {len(base[0][1]): [p for _, p, _ in base]}, {1: [V for _, _, V in base]}
    records = sorted({r for r, _, _ in base})
    paths = []
    for name in ("direct", "graph"):
        ctx = bp.Context(0)
        gens = bp.Gens(ctx, 64, 32)
        if name == "graph":
            ctx._check(bp.lib().bp_rangeproof_verify_reserve(ctx._h, gens._h, 64, 1, count, nb))
        paths.append((name, ctx, gens))
    failing_chunks, kinds, codes = set(), set(), set()
    try:
        for round_ in range(3):
            seed = SEED + 3000 + 100 * nb + round_
            rnd = random.Random(seed)
            j0 = rnd.randrange(len(base))
            items = [[base[(j0 + i) % len(base)][1], base[(j0 + i) % len(base)][2], 64, "valid", base[(j0 + i) % len(base)][0]] for i in range(count * nb)]
            for b in range(nb):
                level = LEVELS[(round_ * nb + b) % 4]
                k = {"none": 0, "one": 1, "few": rnd.randint(2, 4), "many": rnd.randint(5, max(5, min(64, count // 3)))}[level]
                for i in rnd.sample(range(count), k):
                    it = items[b * count + i]
                    if rnd.random() < 0.5:
                        sub = it[:4]; _mutate_rp(rnd, sub, pool, by_len, by_m, resize=False); it[:4] = sub
                        continue
                    kind = rnd.choice(RECORD_MUTATIONS)
                    if kind == "records swapped":
                        o = items[rnd.randrange(count * nb)]
                        if o is it or o[4] == it[4]:
                            continue
                        it[4], o[4] = o[4], it[4]; o[3] = kind
                    elif kind == "another proof's record":
                        it[4] = rnd.choice([r for r in records if r != it[4]])
                    elif kind == "malformed record":
                        it[4] = malformed_record(rnd, rnd.randrange(2))
                    else:
                        r = bytearray(it[4]); r[202] ^= rnd.randrange(1, 256); it[4] = bytes(r)
                    it[3] = kind
                    kinds.add(kind)
            want = _want(orc, og, 64, 1, [(it[4], it[0], it[1]) for it in items])
            codes |= set(want)
            cats = [_rp_category(orc, w, it[0], it[1]) for it, w in zip(items, want)]
            chunks = [len({(i % count) // 32 for i in range(b * count, (b + 1) * count) if cats[i] == "wrong"}) for b in range(nb)]
            failing_chunks |= set(chunks)
            ok_want, dev_want = _expected(want, count, nb, {b for b in range(nb) if chunks[b]})
            triples = [(it[4], it[0], it[1]) for it in items]
            recs, proofs, Vs = b"".join(t for t, _, _ in triples), b"".join(p for _, p, _ in triples), b"".join(V for _, _, V in triples)
            names = [f"batch {i // count} {it[3]}" for i, it in enumerate(items)]
            sd = bytes([round_ + 1]) * 32
            for name, ctx, gens in paths:
                tag = f"test_launch_group_fuzz_with_records[{nb}x{count} {name}]"
                got, ok = bp.verify_group_each(ctx, gens, recs, proofs, Vs, 64, 1, count, nb, seed=sd)
                assert got == want, _diff(tag, seed, round_, names, got, want)
                assert ok == ok_want, f"{tag} seed {seed} round {round_}: flags {ok} want {ok_want} (failing chunks {chunks})"
                dgot, dok = _device_each(bp, ctx, gens, 64, 1, count, nb, triples, sd, front=1)
                assert dgot == dev_want, _diff(tag + " device", seed, round_, names, dgot, dev_want)
                assert dok == ok_want, f"{tag} device seed {seed} round {round_}: flags {dok} want {ok_want} (failing chunks {chunks})"
    finally:
        for _, ctx, gens in paths:
            gens.close(); ctx.close()
    assert 0 in failing_chunks and failing_chunks - {0}, failing_chunks
    if count > 4 * 32:
        assert failing_chunks & {2, 3, 4} and max(failing_chunks) > 4, failing_chunks
    assert kinds == set(RECORD_MUTATIONS), kinds
    assert codes >= {OK, VERIFICATION_ERROR, FORMAT_ERROR}, codes
