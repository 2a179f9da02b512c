"""Batch verifiers against invalid proofs whose errors cancel in the random linear combination.

A batch (or a launch group) is accepted when one combination of every proof's verification equation, each times a per-proof random
weight, vanishes.  Every damage the other tests make leaves one proof's equation nonzero on its own; here each test builds a set of
proofs that are each invalid but differ only in scalars the transcript never absorbs (the inner-product a, b of a range proof or an
R1CS proof, a and r of a LinearProof).  Their challenges are identical and each check is affine in those scalars, so with weights
that did not depend on them the errors would cancel: P with a + d beside P with a - d, or a + d, a + d, a - 2d.  Every test first
asserts that its inputs are that case (the oracle rejects each member, the members differ only in the changed scalar, and their
replayed challenges are byte-identical), and every verdict must equal the oracle's per-proof verdict.

CPU tier: the device's range-proof scalar assembly compiled for the host (tests/host_emul) summed over a cancelling set and checked
with the oracle's MSM; the weight rows of the range-proof and LinearProof replays against a flipped bit of each unabsorbed scalar and
against an independent Python STROBE; the R1CS weight through the mock engine (tests/mock_engine/mock_r1cs.c keeps the challenge
array of its last batch call).
GPU tier: bp.verify_batch, bp.verify_group (direct, graph and device paths), the reject path's chunk level, LinearVerifier and
bp.r1cs_verify_batch, including an R1CS pair built from the weights a known seed gives."""
import ctypes
import json
import os
import random
import subprocess
import sys

import pytest

from oracle_binding import L_ORDER as l
from test_linear_verify_batch import _gens, gpu_proofs, orc_proof, rng_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LABEL = b"AggregateRangeProofBenchmark"
OK, VERIFICATION_ERROR = 0, 1
RP_RAW_C, RP_RAW_RHO, RP_RAW_U = 4, 5, 6
GEOMS = [(8, 1), (64, 1), (16, 4)]
KINDS = ["a+-d", "b+-d", "a triple"]


def le(x, n=32):
    return x.to_bytes(n, "little")


def lg(n):
    return n.bit_length() - 1


def with_scalar(proof: bytes, off: int, delta: int) -> bytes:
    """proof with the canonical scalar at off replaced by (scalar + delta) mod l"""
    v = (int.from_bytes(proof[off:off + 32], "little") + delta) % l
    return proof[:off] + le(v) + proof[off + 32:]


def cancelling_set(proof: bytes, off_a: int, kind: str, d: int):
    """(members, offset of the changed scalar): a +- d, b +- d (b right after a) or a + d, a + d, a - 2d"""
    if kind == "a+-d":
        return [with_scalar(proof, off_a, d), with_scalar(proof, off_a, -d)], off_a
    if kind == "b+-d":
        return [with_scalar(proof, off_a + 32, d), with_scalar(proof, off_a + 32, -d)], off_a + 32
    assert kind == "a triple"
    return [with_scalar(proof, off_a, d), with_scalar(proof, off_a, d), with_scalar(proof, off_a, -2 * d)], off_a


def assert_differs_only_at(members, proof, off):
    for p in members:
        assert len(p) == len(proof) and p[:off] == proof[:off] and p[off + 32:] == proof[off + 32:] and p[off:off + 32] != proof[off:off + 32]


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    e.emul_rp_transcript_both.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32,
                                          ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    e.emul_lin_transcript.restype = ctypes.c_uint32
    return e


# ---------------------------------------------------------------------------------------------------------------------- range proofs
_RP = {}


def rp_case(orc, n, m):
    """one oracle proof at (n, m), its commitments and the points of its verification MSM [B~, B, G.., H.. | A, S, T1, T2, L.., R.., V..]"""
    if (n, m) not in _RP:
        og = orc.gens(n, m)
        rnd = random.Random(100 * n + m)
        rc, pb, vc = orc.rangeproof_prove(og, orc.transcript(LABEL), [rnd.randrange(1 << n) for _ in range(m)],
                                          b"".join(le(rnd.randrange(l)) for _ in range(m)), n, seed=le(7 * n + m))
        assert rc == 0
        k = lg(n * m)
        B, Bb = orc.pedersen()
        pts = [Bb, B] + [orc.gens_get(og, w, j, i) for w in (0, 1) for j in range(m) for i in range(n)]
        pts += [pb[0:32], pb[32:64], pb[64:96], pb[96:128]] + [pb[224 + 64 * j:256 + 64 * j] for j in range(k)] + \
               [pb[256 + 64 * j:288 + 64 * j] for j in range(k)] + [vc[32 * j:32 * j + 32] for j in range(m)]
        _RP[(n, m)] = (og, pb, vc, b"".join(pts))
    return _RP[(n, m)]


def rp_tstate(E):
    st = ctypes.create_string_buffer(203)
    E.emul_transcript_new(LABEL, len(LABEL), st)
    return st.raw


def rp_replay(E, proof, k, V, n, m, tstate, seed):
    """both replay forms: (rows of the byte-wise form, rows of the scheduled form); both must accept and agree"""
    rows = RP_RAW_U + k
    rb, rs = ctypes.create_string_buffer(64 * rows), ctypes.create_string_buffer(64 * rows)
    st = E.emul_rp_transcript_both(proof, k, V, n, m, tstate, seed, rb, rs)
    assert st == 0, st
    assert rb.raw == rs.raw
    return rb.raw


def rp_challenges(raw):
    """the replayed challenge rows without the weight rows C and RHO"""
    return raw[:64 * RP_RAW_C] + raw[64 * RP_RAW_U:]


def assert_rp_adversarial(E, orc, og, members, proof, off, vc, n, m):
    assert_differs_only_at(members, proof, off)
    for p in members:
        assert orc.rangeproof_verify(og, orc.transcript(LABEL), p, vc, m, n) == VERIFICATION_ERROR
    k, ts = lg(n * m), rp_tstate(E)
    assert len({rp_challenges(rp_replay(E, p, k, vc, n, m, ts, bytes(32))) for p in members + [proof]}) == 1


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n,m", GEOMS)
def test_rp_cancelling_set_does_not_vanish_in_the_combination(E, orc, n, m, kind):
    """the device's weighted scalars of each member, summed, against the oracle's MSM: each member alone and the whole set must
    leave a nonzero combination"""
    og, pb, vc, pts = rp_case(orc, n, m)
    k = lg(n * m)
    members, off = cancelling_set(pb, 224 + 64 * k, kind, random.Random(n + 3 * m).randrange(1, l))
    assert_rp_adversarial(E, orc, og, members, pb, off, vc, n, m)
    terms = len(pts) // 32
    ts, seed = rp_tstate(E), bytes(range(32))
    total = [0] * terms
    for p in members:
        out = ctypes.create_string_buffer(32 * terms)
        assert E.emul_rp_scalars(p, k, vc, n, m, ts, seed, out) == 0
        rc, res = orc.msm(out.raw, pts)
        assert rc == 0 and res != bytes(32)
        total = [(t + int.from_bytes(out.raw[32 * i:32 * i + 32], "little")) % l for i, t in enumerate(total)]
    rc, res = orc.msm(b"".join(le(t) for t in total), pts)
    assert rc == 0 and res != bytes(32), "the members' errors cancel in the combination"
    out = ctypes.create_string_buffer(32 * terms)                  # the unchanged proof still gives the identity
    assert E.emul_rp_scalars(pb, k, vc, n, m, ts, seed, out) == 0 and orc.msm(out.raw, pts) == (0, bytes(32))


@pytest.mark.parametrize("n,m", GEOMS)
def test_rp_weights_depend_on_a_and_b(E, orc, n, m):
    """one flipped bit of a or of b: the same challenges, other C and RHO rows, in both replay forms"""
    _, pb, vc, _ = rp_case(orc, n, m)
    k = lg(n * m); ts = rp_tstate(E); seed = bytes([0x5A]) * 32
    base = rp_replay(E, pb, k, vc, n, m, ts, seed)
    for off in (224 + 64 * k, 224 + 64 * k + 32):
        for byte, bit in ((0, 0), (17, 5)):
            q = bytearray(pb); q[off + byte] ^= 1 << bit
            assert int.from_bytes(q[off:off + 32], "little") < l
            raw = rp_replay(E, bytes(q), k, vc, n, m, ts, seed)
            assert rp_challenges(raw) == rp_challenges(base)
            for row in (RP_RAW_C, RP_RAW_RHO):
                assert raw[64 * row:64 * row + 64] != base[64 * row:64 * row + 64], (off, byte, row)


@pytest.mark.parametrize("n,m", GEOMS)
def test_rp_weight_rows_against_python_strobe(E, orc, n, m):
    """the range-proof replay through bp.Transcript (mod.rs:368-393, inner_product_proof.rs:213-222), then the weights with an
    independent Python STROBE: build_rng().rekey_with_witness_bytes("ipp_a_b", a || b).finalize(seed).fill_bytes(128)"""
    import bulletproofs_b200 as bp
    _, pb, vc, _ = rp_case(orc, n, m)
    k = lg(n * m)
    t = bp.Transcript(LABEL)
    ts = t.to_bytes()
    t.append_message(b"dom-sep", b"rangeproof v1"); t.append_u64(b"n", n); t.append_u64(b"m", m)
    for j in range(m):
        t.append_message(b"V", vc[32 * j:32 * j + 32])
    t.append_message(b"A", pb[0:32]); t.append_message(b"S", pb[32:64])
    want = [t.challenge_bytes(b"y", 64), t.challenge_bytes(b"z", 64)]
    t.append_message(b"T_1", pb[64:96]); t.append_message(b"T_2", pb[96:128])
    want.append(t.challenge_bytes(b"x", 64))
    for lab, o in ((b"t_x", 128), (b"t_x_blinding", 160), (b"e_blinding", 192)):
        t.append_message(lab, pb[o:o + 32])
    want.append(t.challenge_bytes(b"w", 64))
    t.append_message(b"dom-sep", b"ipp v1"); t.append_u64(b"n", n * m)
    us = []
    for j in range(k):
        t.append_message(b"L", pb[224 + 64 * j:256 + 64 * j]); t.append_message(b"R", pb[256 + 64 * j:288 + 64 * j])
        us.append(t.challenge_bytes(b"u", 64))
    rnd = random.Random(n * m)
    for seed in (bytes(32), rnd.randbytes(32)):
        raw = rp_replay(E, pb, k, vc, n, m, ts, seed)
        assert [raw[64 * r:64 * r + 64] for r in range(4)] == want
        assert [raw[64 * (RP_RAW_U + j):64 * (RP_RAW_U + j + 1)] for j in range(k)] == us
        ab = pb[224 + 64 * k:224 + 64 * k + 64]
        assert raw[64 * RP_RAW_C:64 * RP_RAW_U] == rng_bytes(t.to_bytes(), seed, 128, b"ipp_a_b", ab)


# ---------------------------------------------------------------------------------------------------------------------- LinearProof
def lin_rows(E, p, n, G, F, B, seed=bytes(32)):
    import bulletproofs_b200 as bp
    k = lg(n)
    raw = ctypes.create_string_buffer(64 * (k + 2))
    assert E.emul_lin_transcript(p.proof, k, n, p.C, p.b, B + F + G, bp.Transcript(p.label).to_bytes(), seed, raw) == OK
    return raw.raw[:64 * (k + 1)], raw.raw[64 * (k + 1):]


def test_linear_weight_depends_on_a_and_r(E, orc):
    n = 16; k = lg(n); G, F, B = _gens(orc, n)
    p = orc_proof(orc, G, F, B, n, 11, b"soundness linear")
    chal, rho = lin_rows(E, p, n, G, F, B)
    for off in (64 * k + 32, 64 * k + 64):                          # a, r
        for byte, bit in ((0, 0), (20, 3)):
            q = bytearray(p.proof); q[off + byte] ^= 1 << bit
            c2, r2 = lin_rows(E, p.replace(proof=bytes(q)), n, G, F, B)
            assert c2 == chal and r2 != rho, (off, byte)


# ---------------------------------------------------------------------------------------------------------------------- R1CS
# The R1CS weight rho is computed on the host (r1cs::verify_batch) and handed to bp_r1cs_verify_batch in its challenge array.  A child
# process runs a batch through the mock engine (the same C ABI on the oracle's CPU arithmetic) and reads that array back.
_MOCK_CHILD = r"""
import ctypes, json, os, sys
root = sys.argv[1]
sys.path[:0] = [root, os.path.join(root, "tests")]
import bulletproofs_b200 as bp
bp.LIB_PATH = os.path.join(root, "tests", "mock_engine", "libmockbpmsm_r1cs.so")
bp.HOST_LIB_PATH = os.path.join(root, "tests", "mock_engine", "libbulletproofs_host_mock_r1cs.so")
req = json.load(sys.stdin)
ctx = bp.Context(0); gens = bp.Gens(ctx, req["cap"], 1)
L = bp.lib(); L.mock_r1cs_last_chal.restype = ctypes.c_size_t; L.mock_r1cs_last_dims.restype = ctypes.c_size_t
out = []
for run in req["runs"]:
    items = [(bp.Transcript(state=bytes.fromhex(t)), g, bytes.fromhex(V), bytes.fromhex(p), par) for t, g, V, p, par in run["items"]]
    codes = bp.r1cs_verify_batch(ctx, gens, items, ext_seed=bytes.fromhex(run["seed"]))
    np_ = L.mock_r1cs_last_dims(None, 0); dims = (ctypes.c_uint32 * (4 * np_))(); L.mock_r1cs_last_dims(dims, 4 * np_)
    nb = L.mock_r1cs_last_chal(None, 0); ch = ctypes.create_string_buffer(nb); L.mock_r1cs_last_chal(ch, nb)
    rho, at = [], 0
    for j in range(np_):
        rho.append(int.from_bytes(ch.raw[32 * (at + 5):32 * (at + 6)], "little")); at += 7 + dims[4 * j].bit_length() - 1
    out.append({"codes": codes, "rho": rho})
gens.close(); ctx.close()
print(json.dumps(out))
"""


def mock_r1cs_weights(runs, cap):
    """runs = [(items, seed)] of test_r1cs_batch.Item; returns [(codes, rho of every proof the host phase sent)] from the mock engine"""
    import bulletproofs_b200 as bp
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_engine"))
    import build_mock_r1cs
    build_mock_r1cs.build()
    req = {"cap": cap, "runs": [{"seed": seed.hex(), "items": [(it.bp_transcript(bp).to_bytes().hex(), it.gadget, it.V.hex(), it.proof.hex(), it.param)
                                                              for it in items]} for items, seed in runs]}
    env = dict(os.environ); env.pop("BP_TEST_MOCK_ENGINE", None); env.pop("BP_TEST_R1CS_MOCK", None)
    r = subprocess.run([sys.executable, "-c", _MOCK_CHILD, ROOT], input=json.dumps(req), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return [(o["codes"], o["rho"]) for o in json.loads(r.stdout.splitlines()[-1])]


def r1cs_base(orc):
    from test_r1cs_batch import range_item
    og = orc.gens(16, 1)
    return og, range_item(orc, og, 10, 1)                           # 10 multipliers, padded_n = 16: four IPP rounds


def r1cs_with(it, name, off, delta):
    return it.replace(name, proof=with_scalar(it.proof, off, delta))


def test_r1cs_weight_depends_on_a_and_b_through_the_mock_engine(orc):
    """the same proof position and seed, only a or only b changed: another rho"""
    og, P = r1cs_base(orc)
    a_off, b_off = len(P.proof) - 64, len(P.proof) - 32
    seed = bytes(range(32))
    variants = [P, r1cs_with(P, "a+1", a_off, 1), r1cs_with(P, "b+1", b_off, 1), r1cs_with(P, "a-5", a_off, -5)]
    res = mock_r1cs_weights([([v], seed) for v in variants], 16)
    assert [codes for codes, _ in res] == [[v.expected(orc, og)] for v in variants] == [[OK]] + [[VERIFICATION_ERROR]] * 3
    rhos = [rho[0] for _, rho in res]
    assert len(set(rhos)) == len(rhos), rhos
    assert mock_r1cs_weights([([P], seed)], 16)[0][1] == [rhos[0]]             # and it is a function of the inputs


# ---------------------------------------------------------------------------------------------------------------------- GPU tier
_WORK = {}


def rp_work(orc, n, m, count):
    """`count` distinct valid oracle proofs at (n, m) and their commitments"""
    if (n, m, count) not in _WORK:
        from test_gpu_parity import _workload
        og = orc.gens(n, m)
        proofs, Vs = _workload(orc, og, LABEL, n, m, count, seed=9000 + n + m)
        _WORK[(n, m, count)] = (og, proofs, Vs, len(proofs) // count)
    return _WORK[(n, m, count)]


def rp_inputs(orc, n, m, total, placed, src=3, kind="a+-d", d=None, extra_bad=()):
    """`total` proofs (16 distinct valid proofs, repeated) with the members of a cancelling set made from proof `src` at the positions
    `placed` (with src's commitments), and a proof whose t_x has one bit flipped at each position of extra_bad"""
    og, proofs, Vs, plen = rp_work(orc, n, m, 16)
    k = lg(n * m)
    reps = (total + 15) // 16
    pb, vb = bytearray((proofs * reps)[:plen * total]), bytearray((Vs * reps)[:32 * m * total])
    P, V = proofs[src * plen:(src + 1) * plen], Vs[32 * m * src:32 * m * (src + 1)]
    members, off = cancelling_set(P, 224 + 64 * k, kind, d or random.Random(total + len(placed)).randrange(1, l))
    assert len(members) == len(placed)
    for i, q in zip(placed, members):
        pb[plen * i:plen * (i + 1)] = q; vb[32 * m * i:32 * m * (i + 1)] = V
    for i in extra_bad:
        pb[plen * i + 128] ^= 1
    want = orc.verify_many(og, orc.transcript(LABEL), bytes(pb), plen, bytes(vb), n, m, total)
    assert [i for i, w in enumerate(want) if w] == sorted(list(placed) + list(extra_bad))
    return og, P, V, members, off, bytes(pb), bytes(vb), plen, want


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n,m", [(64, 1), (16, 4)])
def test_gpu_verify_batch_rejects_cancelling_sets(gpu_ctx, orc, E, n, m, kind):
    import bulletproofs_b200 as bp
    count = 64
    placed = (5, 37, 60) if kind == "a triple" else (5, 37)
    og, P, V, members, off, pb, vb, plen, want = rp_inputs(orc, n, m, count, placed, kind=kind)
    assert_rp_adversarial(E, orc, og, members, P, off, V, n, m)
    gens = bp.Gens(gpu_ctx, n, m)
    for seed in (bytes(32), bytes([0xC3]) * 32, None):
        got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), pb, vb, n, m, count, seed=seed)
        assert got == want, (seed, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w])
    gens.close()


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["split", "one batch"])
def test_gpu_group_rejects_a_cancelling_pair(orc, E, where):
    """4 batches of 24 in one launch group: the pair's halves in batches 1 and 3, or both in batch 2.  Host entry points on the
    direct and graph paths (exact verdicts, the failing batches' flags 0) and the device entry point (flags only)"""
    import bulletproofs_b200 as bp
    from test_gpu_group_check import _check_case
    n, m, count, nb = 64, 1, 24, 4
    placed, failing = ((24 + 5, 3 * 24 + 9), [1, 3]) if where == "split" else ((2 * 24 + 4, 2 * 24 + 20), [2])
    og, P, V, members, off, pb, vb, plen, want = rp_inputs(orc, n, m, count * nb, placed)
    assert_rp_adversarial(E, orc, og, members, P, off, V, n, m)
    got = _check_case(bp, orc, og, n, m, count, nb, bytearray(pb), bytearray(vb), plen, failing=failing)
    assert got == want


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["one chunk", "chunks 0 and 1"])
def test_gpu_reject_path_chunk_level_rejects_a_cancelling_pair(gpu_ctx, orc, E, where):
    """128 proofs (4 chunks of 32) with an ordinary bad proof in chunk 3 so that the batch check fails and the reject path's first
    level re-checks each chunk with the same weights; two failing chunks, so the second level runs on those chunks only.  The pair
    inside chunk 1 must make that chunk fail; split across chunks 0 and 1 (the control) each half fails its chunk on its own."""
    import bulletproofs_b200 as bp
    assert E.emul_rp_chunk() == 32 and not E.emul_rp_recheck_whole_batch(3)
    n, m, count = 64, 1, 128
    placed = (40, 50) if where == "one chunk" else (10, 40)
    og, P, V, members, off, pb, vb, plen, want = rp_inputs(orc, n, m, count, placed, extra_bad=(100,))
    assert_rp_adversarial(E, orc, og, members, P, off, V, n, m)
    gens = bp.Gens(gpu_ctx, n, m)
    got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), pb, vb, n, m, count, seed=bytes(range(32)))
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    gens.close()


@pytest.mark.gpu
@pytest.mark.parametrize("scalar", ["r", "a"])
def test_gpu_linear_verify_batch_rejects_a_cancelling_pair(gpu_ctx, orc, E, scalar):
    import bulletproofs_b200 as bp
    n = 16; k = lg(n)
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 40)
    G, F, B = gfb
    src = proofs[7]
    off = 64 * k + (64 if scalar == "r" else 32)
    d = random.Random(off).randrange(1, l)
    pair = [src.replace(proof=with_scalar(src.proof, off, s * d)) for s in (1, -1)]
    assert_differs_only_at([p.proof for p in pair], src.proof, off)
    assert len({lin_rows(E, p, n, G, F, B)[0] for p in pair + [src]}) == 1
    items = proofs[:7] + [pair[0]] + proofs[8:30] + [pair[1]] + proofs[31:]
    want = [orc.linear_verify(orc.transcript(p.label), p.proof, p.C, G, F, B, p.b) for p in items]
    assert [i for i, w in enumerate(want) if w] == [7, 30] and want[7] == want[30] == VERIFICATION_ERROR
    V = bp.LinearVerifier(gpu_ctx, G, F, B)
    for seed in (bytes(32), None):
        assert V.verify_batch([p.item(bp) for p in items], seed=seed) == want, seed
    V.close()


@pytest.mark.gpu
def test_gpu_r1cs_rejects_cancelling_pairs(gpu_ctx, orc):
    """an a + d, a - d pair (each position finalises with its own external bytes), and a pair a + d1, a + d2 with d2 = -d1 rho1 / rho2
    built from the weights the public seed gives to the unchanged proof at those positions"""
    import bulletproofs_b200 as bp
    from test_r1cs_batch import check_batch
    og, P = r1cs_base(orc)
    a_off = len(P.proof) - 64
    seed = bytes(range(32))
    (codes, rho), = mock_r1cs_weights([([P, P, P], seed)], 16)
    assert codes == [OK] * 3 and len(rho) == 3
    d1 = random.Random(5).randrange(1, l)
    d2 = -d1 * rho[0] * pow(rho[1], l - 2, l) % l
    gens = bp.Gens(gpu_ctx, 16, 1)
    for name, (e1, e2) in (("equal d", (d1, -d1)), ("known seed", (d1, d2))):
        pair = [r1cs_with(P, f"{name} 1", a_off, e1), r1cs_with(P, f"{name} 2", a_off, e2)]
        assert_differs_only_at([it.proof for it in pair], P.proof, a_off)
        items = pair + [P]
        assert [it.expected(orc, og) for it in items] == [VERIFICATION_ERROR, VERIFICATION_ERROR, OK]
        assert check_batch(bp, gpu_ctx, gens, orc, og, items, seed=seed) == [VERIFICATION_ERROR, VERIFICATION_ERROR, OK], name
    gens.close()
