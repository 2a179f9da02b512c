"""GPU tier (-m gpu): seeded mutation fuzzing of the batch verifiers whose proofs come from outside the program -- bp.verify_mixed, the
launch groups (verify_group on the direct and on the graph path, run_device), bp.r1cs_verify_batch and LinearVerifier.verify_batch --
against the oracle's verdict of each item alone.

One mutation engine works on a per-type field layout (32-byte point and scalar fields, the R1CS version byte): bit flips, byte stomps,
swapped fields, another proof under this item's commitments, 0 / 0xff / l - 1 / l / p - 1 / p + 1 in a field, truncation and extension
by 1, 32 and 64 bytes, and per type: whole proofs of another geometry or circuit of the same length, another item's commitments or C, the
R1CS version byte, IPP rounds removed or added, another circuit's transcript, non-fresh LinearProof transcripts.  Every item records the
mutation it received; a failing verdict names the test, seed, round, item, mutation, got and want, and reproduces from its seed.  Each
test asserts that its inputs reached the verdict codes and the reject-path branches it is about.

CPU tier: the R1CS fuzz through the mock engine (tests/mock_engine: the host mirror on the oracle's arithmetic), as
test_r1cs_batch.py's tests run there, so that a failure under both points at the host mirror and a GPU-only failure at the device."""
import os
import random
import subprocess
import sys

import pytest

from oracle_binding import L_ORDER as l, P_FIELD as p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# BP_TEST_R1CS_MOCK=1 (set only by test_r1cs_fuzz_through_the_mock_engine for its child process): the Python binding and the C++ host
# mirror run against tests/mock_engine/libmockbpmsm_r1cs.so, the mock engine with bp_r1cs_verify_batch (tests/mock_engine/mock_r1cs.c)
if os.environ.get("BP_TEST_R1CS_MOCK") == "1":
    import bulletproofs_b200 as _bp
    _bp.LIB_PATH = os.path.join(ROOT, "tests", "mock_engine", "libmockbpmsm_r1cs.so")
    _bp.HOST_LIB_PATH = os.path.join(ROOT, "tests", "mock_engine", "libbulletproofs_host_mock_r1cs.so")

from test_gpu_geometry import GRID, _cell                                          # noqa: E402
from test_gpu_group_check import LABEL, _device_run, _expected                     # noqa: E402
from test_gpu_parity import _workload                                              # noqa: E402
from test_linear_verify_batch import _gens, _secret                                # noqa: E402
from test_r1cs_batch import E, example_item, r1cs_slice, range_item, shuffle_item  # noqa: E402,F401 (E: fixture)

OK, VERIFICATION_ERROR, FORMAT_ERROR, INVALID_BITSIZE, INVALID_GENERATORS_LENGTH = 0, 1, 2, 3, 4
SEED = 20261016
POINT, SCALAR = "point", "scalar"


def le(x, n=32):
    return x.to_bytes(n, "little")


def _diff(test, seed, round_, names, got, want):
    bad = [f"item {i} ({names[i]}): got {g} want {w}" for i, (g, w) in enumerate(zip(got, want)) if g != w]
    more = f" (+{len(bad) - 8} more)" if len(bad) > 8 else ""
    return f"{test} seed {seed} round {round_}: " + "; ".join(bad[:8]) + more


# ---------------------------------------------------------------------------------------------------------------------- mutation engine
def rp_fields(plen):
    """RangeProof::to_bytes: A, S, T_1, T_2, t_x, t_x_blinding, e_blinding, (L_j, R_j) for k rounds, a, b"""
    k = (plen // 32 - 9) // 2
    return ([(32 * i, POINT) for i in range(4)] + [(128 + 32 * i, SCALAR) for i in range(3)] + [(224 + 32 * j, POINT) for j in range(2 * k)]
            + [(224 + 64 * k, SCALAR), (256 + 64 * k, SCALAR)])


def r1cs_fields(proof):
    """R1CSProof::to_bytes: version byte, 8 points (11 with version 1), t_x, t_x_blinding, e_blinding, the IPP's (L_j, R_j), a, b"""
    pts, nf = (11 if proof[0] == 1 else 8), (len(proof) - 1) // 32
    kind = lambda f: POINT if f < pts or pts + 3 <= f < nf - 2 else SCALAR     # noqa: E731
    return [(1 + 32 * f, kind(f)) for f in range(nf)]


def lin_fields(plen):
    """LinearProof::to_bytes: (L_j, R_j) for k rounds, S, a, r"""
    k = (plen // 32 - 3) // 2
    return [(32 * f, POINT) for f in range(2 * k + 1)] + [(64 * k + 32, SCALAR), (64 * k + 64, SCALAR)]


VALUES = {"zero": bytes(32), "0xff": b"\xff" * 32, "l - 1": le(l - 1), "p - 1": le(p - 1), "l": le(l), "p + 1": le(p + 1)}
KEEP_LENGTH = ("bit flip", "byte stomp", "field swap", "another proof") + tuple(VALUES)
RESIZE = ("truncate", "extend")
R1CS_STRUCTURE = ("version flip", "IPP round removed", "IPP round added")


def mutate(rnd, proof, fields, others=(), kinds=KEEP_LENGTH):
    """(mutated proof, what was done): one mutation of `kinds`; `others` are proofs that may replace this one whole"""
    kind = rnd.choice(kinds)
    b = bytearray(proof)
    others = [q for q in others if q != proof and len(q) == len(proof)]
    if kind == "another proof" and others:
        return rnd.choice(others), "another proof's bytes"
    if kind in ("bit flip", "another proof"):
        i, bit = rnd.randrange(len(b)), rnd.randrange(8)
        b[i] ^= 1 << bit
        return bytes(b), f"bit {bit} of byte {i} flipped"
    if kind == "byte stomp":
        i, v = rnd.randrange(len(b)), rnd.randrange(256)
        b[i] = v
        return bytes(b), f"byte {i} = {v}"
    if kind == "field swap":
        (o1, t1), (o2, t2) = rnd.sample(fields, 2)
        b[o1:o1 + 32], b[o2:o2 + 32] = proof[o2:o2 + 32], proof[o1:o1 + 32]
        return bytes(b), f"{t1} at {o1} swapped with {t2} at {o2}"
    if kind in VALUES:
        o, t = rnd.choice(fields)
        b[o:o + 32] = VALUES[kind]
        return bytes(b), f"{kind} in the {t} at {o}"
    if kind == "truncate":
        d = rnd.choice((1, 32, 64))
        return proof[:-d], f"truncated by {d}"
    if kind == "extend":
        d = rnd.choice((1, 32, 64))
        return proof + rnd.randbytes(d), f"extended by {d}"
    if kind == "version flip":
        b[0] ^= 1
        return bytes(b), "version byte flipped"
    # an IPP round of an R1CS proof: the (L, R) pairs lie between e_blinding and the final a, b
    ipp0 = 1 + 32 * ((11 if proof[0] == 1 else 8) + 3)
    rounds = (len(proof) - 64 - ipp0) // 64
    if kind == "IPP round removed" and rounds:
        return proof[:-128] + proof[-64:], "last IPP round removed"
    pair = proof[ipp0:ipp0 + 64] if rounds else proof[1:65]
    return proof[:-64] + pair + proof[-64:], "an IPP round added"


# ---------------------------------------------------------------------------------------------------------------------- range proofs
def _rp_admitted(plen, n, m, gens_cap=64, gens_parties=32):
    """the (n, m) class a mixed call puts the item in, or None when its parameters decide it (rp_param_verdict)"""
    if plen % 32 or plen < 7 * 32:
        return None
    ne = (plen - 7 * 32) // 32
    if ne < 2 or (ne - 2) % 2 or (ne - 2) // 2 >= 32:
        return None
    if n not in (8, 16, 32, 64) or n > gens_cap or m > gens_parties or m == 0 or n * m != 1 << (ne - 2) // 2:
        return None
    return (n, m)


def _rp_category(orc, code, proof, V):
    """what a verdict means for the combined check: 'valid', 'format' (FormatError), 'excluded' (VerificationError before the MSM:
    a point that does not decode, or an identity A, S, T_1, T_2, L_j or R_j, which the transcript refuses), 'wrong' (VerificationError of
    a proof inside the combination: its chunk fails) or the parameter code"""
    if code == OK:
        return "valid"
    if code == FORMAT_ERROR:
        return "format"
    if code != VERIFICATION_ERROR:
        return f"code {code}"
    pts = [proof[o:o + 32] for o, t in rp_fields(len(proof)) if t == POINT]
    if bytes(32) in pts or not all(orc.point_is_valid(q) for q in pts + [V[i:i + 32] for i in range(0, len(V), 32)]):
        return "excluded"
    return "wrong"


# ---------------------------------------------------------------------------------------------------------------------- 1. mixed call
MIX_CELLS = [(n, m) for n, m in GRID if 16 <= n * m <= 1024]        # every cell with another cell of its proof length, but (64, 32)
ALIASES = [(a, b) for a in MIX_CELLS for b in MIX_CELLS if a != b and a[0] * a[1] == b[0] * b[1]]


def test_mixed_fuzz_cells_cover_every_alias_pair():
    """every pair of grid cells with one proof length, except (64, 32)'s which has none, is submitted as the other"""
    assert len(MIX_CELLS) >= 8 and len(ALIASES) == 2 * (1 + 3 + 6 + 6 + 6 + 3 + 1)
    assert {(n, m) for n, m in GRID if any((n, m) in pair for pair in ALIASES)} == set(MIX_CELLS)


def _mutate_rp(rnd, it, pool, by_len, by_m, resize=True):
    """one mutation of a range-proof item [proof, V, n, name] (in place)"""
    pr, V, n, _ = it
    m, r = len(V) // 32, rnd.random()
    if r < 0.12:
        it[1] = rnd.choice([v for v in by_m[m] if v != V] or [bytes(32) * m]); it[3] = "another item's commitments"
    elif r < 0.22:
        i, bit = rnd.randrange(len(V)), rnd.randrange(8)
        v = bytearray(V); v[i] ^= 1 << bit; it[1] = bytes(v); it[3] = f"bit {bit} of commitment byte {i} flipped"
    elif r < 0.3 and resize:
        (n0, m0), (n1, m1) = rnd.choice([(a, b) for a, b in ALIASES if b[0] * b[1] == n * m])
        it[0] = rnd.choice(pool[(n1, m1)])[0]; it[3] = f"a ({n1},{m1}) proof of the same length"
    else:
        it[0], it[3] = mutate(rnd, pr, rp_fields(len(pr)), by_len[len(pr)], KEEP_LENGTH + (RESIZE if resize else ()))


def _interleave(rnd, a, b):
    """a and b merged at random, each in its own order"""
    out, i, j = [], 0, 0
    while i < len(a) or j < len(b):
        if j == len(b) or (i < len(a) and rnd.random() < len(a) / (len(a) + len(b))):
            out.append(a[i]); i += 1
        else:
            out.append(b[j]); j += 1
    return out


@pytest.mark.gpu
def test_mixed_call_fuzz(gpu_ctx, orc):
    """rounds of ~120 items from every aliasing cell, a third mutated, length-aliased proofs of another geometry next to genuine proofs
    of their class, parameter codes in the odd rounds; a last round with 192 proofs of (64, 1) whose wrong proofs sit in more than four
    of its chunks beside three classes that pass.  Every verdict == the oracle's and bp.verify_batch's for the item alone"""
    import bulletproofs_b200 as bp
    og, ot = orc.gens(64, 32), orc.transcript(LABEL)
    gens = bp.Gens(gpu_ctx, 64, 32)
    pool, by_len, by_m = {}, {}, {}
    for n, m in MIX_CELLS:
        proofs, Vs, plen = _cell(orc, og, n, m)
        pool[(n, m)] = [(proofs[i * plen:(i + 1) * plen], Vs[32 * m * i:32 * m * (i + 1)]) for i in range(4)]
        by_len.setdefault(plen, []).extend(q for q, _ in pool[(n, m)]); by_m.setdefault(m, []).extend(v for _, v in pool[(n, m)])
    alone = {}

    def verdict(pr, V, n):
        if (pr, V, n) not in alone:
            m = len(V) // 32
            ref = orc.rangeproof_verify(og, ot, pr, V, m, n)
            dev = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), pr, V, n, m, 1, proof_len=len(pr), seed=bytes([7]) * 32)[0]
            assert dev == ref, f"verify_batch of one item: ({n},{m}) length {len(pr)} got {dev} want {ref}"
            alone[(pr, V, n)] = ref
        return alone[(pr, V, n)]

    order = ALIASES[:]
    random.Random(SEED).shuffle(order)
    codes, mixed_chunk, whole_class = set(), False, False
    try:
        for round_ in range(5):
            seed = SEED + round_
            rnd = random.Random(seed)
            if round_ < 4:
                items = [[*rnd.choice(pool[c]), c[0], "valid"] for c in (rnd.choice(MIX_CELLS) for _ in range(96))]
                for (n0, m0), (n, m) in order[round_::4]:
                    pr, V = rnd.choice(pool[(n0, m0)])
                    items.append([pr, (V * (m // m0 + 1))[:32 * m], n, f"a ({n0},{m0}) proof as ({n},{m})"])
                    assert verdict(*items[-1][:3]) == VERIFICATION_ERROR, items[-1][3]
                for it in rnd.sample(items, len(items) // 3):
                    _mutate_rp(rnd, it, pool, by_len, by_m)
                if round_ % 2:
                    (p82, V82), (p84, V84) = pool[(8, 2)][0], pool[(8, 4)][1]
                    items += [[p82, V82, 12, "n = 12"], [p82, V82 * 20, 8, "m = 40 above the table's parties"], [p84, V84[:96], 8, "m = 3"]]
                rnd.shuffle(items)
            else:                           # one class of 192 proofs with a wrong proof (t_x + 1) in 5 of its 6 chunks, 3 passing classes
                big = [[*pool[(64, 1)][i % 4], 64, "valid"] for i in range(192)]
                for ch in rnd.sample(range(6), 5):
                    it = big[32 * ch + rnd.randrange(32)]
                    q = bytearray(it[0]); q[128] ^= 1; it[0], it[3] = bytes(q), "t_x + 1"
                for it in rnd.sample(big, 64):
                    _mutate_rp(rnd, it, pool, by_len, by_m)
                rest = [[*pool[c][i % 4], c[0], "valid"] for c in ((8, 4), (32, 4), (16, 16)) for i in range(33)]
                rnd.shuffle(rest)
                items = _interleave(rnd, big, rest)
            got = bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), [tuple(it[:3]) for it in items], seed=bytes([round_]) * 32)
            want = [verdict(*it[:3]) for it in items]
            assert got == want, _diff("test_mixed_call_fuzz", seed, round_, [it[3] for it in items], got, want)
            codes |= set(want)
            classes = {}
            for it, w in zip(items, want):
                cls = _rp_admitted(len(it[0]), it[2], len(it[1]) // 32)
                if cls is not None:
                    classes.setdefault(cls, []).append(_rp_category(orc, w, it[0], it[1]))
            for cls, cats in classes.items():
                chunks = [set(cats[c:c + 32]) for c in range(0, len(cats), 32)]
                mixed_chunk |= any({"format", "excluded", "wrong"} <= ch for ch in chunks)
                if len(cats) >= 160 and sum("wrong" in ch for ch in chunks) > 4:
                    whole_class |= any(set(o) == {"valid"} for c, o in classes.items() if c != cls)
    finally:
        gens.close()
    assert codes >= {OK, VERIFICATION_ERROR, FORMAT_ERROR, INVALID_BITSIZE, INVALID_GENERATORS_LENGTH}, codes
    assert mixed_chunk, "no chunk held a FormatError, an undecodable and a wrong proof together"
    assert whole_class, "no class of 160 proofs or more had more than four failing chunks beside a passing class"


# ---------------------------------------------------------------------------------------------------------------------- 2. launch groups
GROUPS = [(2, 1024), (5, 40), (8, 24)]             # (batches, proofs per batch) of (64, 1)
LEVELS = ("none", "one", "few", "many")


@pytest.mark.gpu
def test_launch_group_fuzz(orc):
    """mutations in random batches of launch groups, so that batches have 0, 1, 2-4 and more than 4 failing chunks of 32: verify_group
    on a context that never reserved the geometry (direct launches) and on one that did (graph replay) give the oracle's verdicts and
    the per-batch flags; run_device on both gives the flags and VerificationError for every well-formed proof of a failing batch"""
    import bulletproofs_b200 as bp
    n, m = 64, 1
    og, ot = orc.gens(n, m), orc.transcript(LABEL)
    proofs, Vs = _workload(orc, og, LABEL, n, m, 24, seed=7100)
    plen = len(proofs) // 24
    base = [(proofs[i * plen:(i + 1) * plen], Vs[32 * i:32 * (i + 1)]) for i in range(24)]
    pool = {(n, m): base}
    by_len, by_m = {plen: [q for q, _ in base]}, {1: [v for _, v in base]}
    alone = {(q, v): OK for q, v in base}
    assert orc.verify_many(og, ot, proofs, plen, Vs, n, m, 24) == [OK] * 24
    failing_chunks = set()
    for nb, count in GROUPS:
        paths = []
        for name in ("direct", "graph"):
            ctx = bp.Context(0)
            gens = bp.Gens(ctx, n, m)
            if name == "graph":
                bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), n, m, count, nb)         # reserve: verify_group replays the graph
            paths.append((name, ctx, gens))
        try:
            for round_ in range(3):
                seed = SEED + 1000 * nb + round_
                rnd = random.Random(seed)
                items = [[*base[i % 24], n, "valid"] for i in range(count * nb)]
                for b in range(nb):
                    level = LEVELS[(round_ * nb + b) % 4]
                    k = {"none": 0, "one": 1, "few": rnd.randint(2, 4), "many": rnd.randint(5, max(5, min(64, count // 3)))}[level]
                    for i in rnd.sample(range(count), k):
                        _mutate_rp(rnd, items[b * count + i], pool, by_len, by_m, resize=False)
                want = []
                for pr, V, _, _ in items:
                    if (pr, V) not in alone:
                        alone[(pr, V)] = orc.rangeproof_verify(og, ot, pr, V, m, n)
                    want.append(alone[(pr, V)])
                cats = [_rp_category(orc, w, it[0], it[1]) for it, w in zip(items, want)]
                chunks = [len({(i % count) // 32 for i in range(b * count, (b + 1) * count) if cats[i] == "wrong"}) for b in range(nb)]
                failing_chunks |= set(chunks)
                ok_want, dev_want = _expected(want, count, nb, {b for b in range(nb) if chunks[b]})
                pb, vb = b"".join(it[0] for it in items), b"".join(it[1] for it in items)
                names = [f"batch {i // count} {it[3]}" for i, it in enumerate(items)]
                for name, ctx, gens in paths:
                    tag = f"test_launch_group_fuzz[{nb}x{count} {name}]"
                    got, ok = bp.verify_group(ctx, gens, bp.Transcript(LABEL), pb, vb, n, m, count, nb, seed=bytes([round_ + 1]) * 32)
                    assert got == want, _diff(tag, seed, round_, names, got, want)
                    assert ok == ok_want, f"{tag} seed {seed} round {round_}: flags {ok} want {ok_want} (failing chunks {chunks})"
                    dgot, dok = _device_run(bp, ctx, gens, n, m, count, nb, pb, vb, bytes([round_ + 1]) * 32)
                    assert dgot == dev_want, _diff(tag + " run_device", seed, round_, names, dgot, dev_want)
                    assert dok == ok_want, f"{tag} run_device seed {seed} round {round_}: flags {dok} want {ok_want} (failing chunks {chunks})"
        finally:
            for _, ctx, gens in paths:
                gens.close(); ctx.close()
    # batches with no failing chunk, with one (first level: chunk then proofs), 2-4 (first level) and more than 4 (second level)
    assert {0, 1} <= failing_chunks and failing_chunks & {2, 3, 4} and max(failing_chunks) > 4, failing_chunks


# ---------------------------------------------------------------------------------------------------------------------- 3. R1CS batches
def _r1cs_pool(orc, og):
    """valid proofs: shuffles with k in {1, 2, 5, 8, 42} (two proofs of k = 2 and 8), the example gadget, range gadgets with n = 10
    (two proofs) and 63"""
    return ([shuffle_item(orc, og, k, 100 + k) for k in (1, 2, 5, 8, 42)] + [shuffle_item(orc, og, k, 200 + k) for k in (2, 8)]
            + [example_item(orc, og), range_item(orc, og, 10, 1), range_item(orc, og, 10, 3), range_item(orc, og, 63, 2)])


def _mutate_r1cs(rnd, it, pool):
    """one mutated copy of R1CS item `it`"""
    r = rnd.random()
    if r < 0.1:
        same = [q for q in pool if len(q.V) == len(it.V) and q.V != it.V]
        if same:
            q = rnd.choice(same)
            return it.replace(f"{it.name} with the commitments of {q.name}", V=q.V)
        i = rnd.randrange(len(it.V)); v = bytearray(it.V); v[i] ^= 1 << rnd.randrange(8)
        return it.replace(f"{it.name} with commitment byte {i} changed", V=bytes(v))
    if r < 0.2:
        q = rnd.choice([q for q in pool if q.name != it.name])
        return it.replace(f"{it.name} with the proof of {q.name}", proof=q.proof)
    if r < 0.27:
        q = rnd.choice([q for q in pool if (q.label, q.k) != (it.label, it.k)])
        return it.replace(f"{it.name} under the transcript of {q.name}", label=q.label, k=q.k if q.k else it.k + 1)
    if r < 0.3 and it.gadget != 0:
        param = rnd.choice([q.param for q in pool if q.gadget == it.gadget and q.param != it.param] or [it.param + 1])
        return it.replace(f"{it.name} with param {param}", param=param)
    kinds = KEEP_LENGTH + RESIZE + R1CS_STRUCTURE * 2
    proof, what = mutate(rnd, it.proof, r1cs_fields(it.proof), [q.proof for q in pool], kinds)
    return it.replace(f"{it.name}: {what}", proof=proof)


def _r1cs_round(bp, ctx, gens, orc, og, test, seed, round_, items, verdicts):
    got = bp.r1cs_verify_batch(ctx, gens, [it.batch_item(bp) for it in items], ext_seed=bytes([round_]) * 32)
    want = []
    for it in items:
        key = (it.label, it.k, it.gadget, it.V, it.proof, it.param)
        if key not in verdicts:
            verdicts[key] = it.expected(orc, og)
        want.append(verdicts[key])
    assert got == want, _diff(test, seed, round_, [it.name for it in items], got, want)
    return want


@pytest.mark.gpu
def test_r1cs_batch_fuzz(gpu_ctx, orc):
    """batches of 30-300 shuffles, example and range gadgets, a third mutated: the field mutations, the version byte flipped (8 points
    read as 11 or the reverse), an IPP round removed or added (the proof parses, lg_n no longer matches padded_n), another circuit's
    proof (another padded_n), commitments, transcript or parameter"""
    import bulletproofs_b200 as bp
    gens, og = bp.Gens(gpu_ctx, 128, 1), orc.gens(128, 1)
    pool, verdicts, codes, kinds = _r1cs_pool(orc, og), {}, set(), set()
    try:
        for round_, size in enumerate((30, 300, 97, 211)):
            seed = SEED + 2000 + round_
            rnd = random.Random(seed)
            items = [rnd.choice(pool) for _ in range(size)]
            for i in rnd.sample(range(size), size // 3):
                items[i] = _mutate_r1cs(rnd, items[i], pool)
            codes |= set(_r1cs_round(bp, gpu_ctx, gens, orc, og, "test_r1cs_batch_fuzz", seed, round_, items, verdicts))
            kinds |= {k for it in items for k in ("version byte", "IPP round removed", "IPP round added", "the proof of", "the transcript of") if k in it.name}
    finally:
        gens.close()
    assert codes >= {OK, VERIFICATION_ERROR, FORMAT_ERROR}, codes
    assert len(kinds) == 5, kinds


@pytest.mark.gpu
def test_r1cs_batch_fuzz_past_one_reject_slice_2049(gpu_ctx, orc, E):
    """one batch of 560 mutated items around a 2049-input shuffle (padded_n = 4096): the reject path re-checks it in two slices"""
    import bulletproofs_b200 as bp
    count = 560
    per = r1cs_slice(E, count, 4096)
    assert per < count, per
    gens, og = bp.Gens(gpu_ctx, 4096, 1), orc.gens(4096, 1)
    pool = _r1cs_pool(orc, og)
    seed = SEED + 2100
    rnd = random.Random(seed)
    items = [rnd.choice(pool) for _ in range(count)]
    for i in rnd.sample(range(count), count // 3):
        items[i] = _mutate_r1cs(rnd, items[i], pool)
    items[per + 7] = shuffle_item(orc, og, 2049, 300)
    try:
        want = _r1cs_round(bp, gpu_ctx, gens, orc, og, "test_r1cs_batch_fuzz_past_one_reject_slice_2049", seed, 0, items, {})
    finally:
        gens.close()
    assert want[per + 7] == OK and VERIFICATION_ERROR in want[:per] and VERIFICATION_ERROR in want[per:]


def test_r1cs_fuzz_through_the_mock_engine(built):
    """test_r1cs_batch_fuzz against the mock engine"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_engine"))
    import build_mock_r1cs
    build_mock_r1cs.build()
    env = dict(os.environ, BP_TEST_R1CS_MOCK="1")
    env.pop("BP_TEST_MOCK_ENGINE", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_verifier_fuzz.py", "-m", "gpu", "-q", "-k", "r1cs and not 2049", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    tail = "\n".join(r.stdout.splitlines()[-15:])
    assert r.returncode == 0, tail + r.stderr[-2000:]
    assert int(tail.split(" passed")[0].split()[-1]) == 1, tail


# ---------------------------------------------------------------------------------------------------------------------- 4. LinearProof batches
LIN_LABEL = b"linear fuzz"
LIN_CALLERS = (b"application prefix", b"session id")
LIN_LENGTHS = (0, 1, 7, 100, 137, 150, 163)


def _lin_states(orc):
    """caller transcripts: LIN_LABEL, then append_message(caller label, message) of every length in LIN_LENGTHS (oracle states)"""
    return [orc.transcript_append(orc.transcript(LIN_LABEL), c, bytes(range(n))) for c in LIN_CALLERS for n in LIN_LENGTHS]


def test_linear_caller_states_reach_the_rate():
    """the STROBE position (byte 200 of the wire state) of the caller transcripts: one state leaves the verifier's first header
    straddling the 166-byte rate (position 165), one its first operation (header, "dom-sep", length) and several wrapped inside the
    caller's own append"""
    from oracle_binding import Oracle
    orc = Oracle()
    pos = [st[200] for st in _lin_states(orc)]
    fresh = orc.transcript(LIN_LABEL)[200]
    starts = [orc.transcript(LIN_LABEL)[200] + 8 + len(c) + n for c in LIN_CALLERS for n in LIN_LENGTHS]
    assert 165 in pos and any(166 - 13 <= q < 165 for q in pos), pos
    assert sum(s >= 166 for s in starts) >= 4 and all(q == s % 166 for q, s in zip(pos, starts) if s < 2 * 166), (fresh, pos)


_LIN = {}


def _lin_valid(orc, n):
    """two valid proofs at n under each caller state, made by orc.linear_create under that state: [(state, proof, C, b)]"""
    if n not in _LIN:
        G, F, B = _gens(orc, n)
        out = []
        for s, st in enumerate(_lin_states(orc)):
            for j in range(2):
                a, b, r = _secret(n, 100000 * n + 10 * s + j)
                rc, C = orc.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % l), G + B + F)
                assert rc == 0
                rc, _, proof = orc.linear_create(st, le(10 * s + j), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), G, F, B)
                assert rc == 0
                out.append((st, proof, C, b"".join(map(le, b))))
        _LIN[n] = out
    return _LIN[n]


def _mutate_lin(rnd, it, valid, n):
    """(mutated copy of [state, proof, C, b], what was done)"""
    st, proof, C, b = it
    r = rnd.random()
    if r < 0.1:
        return (st, proof, rnd.choice([q[2] for q in valid if q[2] != C]), b), "another item's C"
    if r < 0.17:
        i, bit = rnd.randrange(32), rnd.randrange(8)
        c = bytearray(C); c[i] ^= 1 << bit
        return (st, proof, bytes(c), b), f"bit {bit} of C byte {i} flipped"
    if r < 0.32:
        i = rnd.randrange(n)
        x = int.from_bytes(b[32 * i:32 * i + 32], "little")
        v, what = rnd.choice([(rnd.randrange(l), "random"), (x ^ 1 if x ^ 1 < l else x - 1, "x +- 1"), (0, "0"), (l - 1, "l - 1"),
                              (int.from_bytes(rnd.choice(valid)[3][32 * i:32 * i + 32], "little"), "another item's")])
        return (st, proof, C, b[:32 * i] + le(v) + b[32 * i + 32:]), f"b_{i} = {what}"
    if r < 0.4:
        return (rnd.choice([q[0] for q in valid if q[0] != st]), proof, C, b), "another caller state"
    if r < 0.44:
        return (None, proof, C, b), "a fresh transcript"
    q, what = mutate(rnd, proof, lin_fields(len(proof)), [q[1] for q in valid], KEEP_LENGTH)
    return (st, q, C, b), what


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 64, 256])
def test_linear_batch_fuzz(gpu_ctx, orc, n):
    """batches of up to 300 proofs under non-fresh caller transcripts (some at the rate), a third mutated in the proof bytes, C, one
    entry of b (canonical values) or the caller state"""
    import bulletproofs_b200 as bp
    G, F, B = _gens(orc, n)
    valid = _lin_valid(orc, n)
    fresh = orc.transcript(LIN_LABEL)
    V = bp.LinearVerifier(gpu_ctx, G, F, B)
    verdicts, codes = {}, set()
    try:
        for round_, count in enumerate((57, 300)):
            seed = SEED + 3000 + 10 * n + round_
            rnd = random.Random(seed)
            items = [(valid[i % len(valid)], "valid") for i in rnd.sample(range(max(count, len(valid))), count)]
            for i in rnd.sample(range(count), count // 3):
                items[i] = _mutate_lin(rnd, items[i][0], valid, n)
            items = [((fresh if st is None else st, pr, C, b), what) for (st, pr, C, b), what in items]
            got = V.verify_batch([(bp.Transcript(state=st[:bp.TRANSCRIPT_BYTES]), pr, C, b) for (st, pr, C, b), _ in items], seed=bytes([round_]) * 32)
            want = []
            for it, _ in items:
                if it not in verdicts:
                    verdicts[it] = orc.linear_verify(it[0], it[1], it[2], G, F, B, it[3])
                want.append(verdicts[it])
            assert got == want, _diff(f"test_linear_batch_fuzz[{n}]", seed, round_, [w for _, w in items], got, want)
            codes |= set(want)
    finally:
        V.close()
    assert codes == {OK, VERIFICATION_ERROR, FORMAT_ERROR}, codes


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 64])
def test_linear_batch_under_caller_transcripts_at_the_rate(gpu_ctx, orc, n):
    """valid proofs made under caller transcripts at every position of LIN_LENGTHS, the rate-crossing ones included, verify in one batch;
    the same proofs under fresh transcripts are rejected"""
    import bulletproofs_b200 as bp
    G, F, B = _gens(orc, n)
    valid = _lin_valid(orc, n)
    V = bp.LinearVerifier(gpu_ctx, G, F, B)
    try:
        assert V.verify_batch([(bp.Transcript(state=st[:bp.TRANSCRIPT_BYTES]), pr, C, b) for st, pr, C, b in valid], seed=bytes(32)) == [OK] * len(valid)
        fresh = orc.transcript(LIN_LABEL)
        assert [orc.linear_verify(fresh, pr, C, G, F, B, b) for _, pr, C, b in valid] == [VERIFICATION_ERROR] * len(valid)
        assert V.verify_batch([(bp.Transcript(LIN_LABEL), pr, C, b) for _, pr, C, b in valid], seed=bytes(32)) == [VERIFICATION_ERROR] * len(valid)
    finally:
        V.close()
