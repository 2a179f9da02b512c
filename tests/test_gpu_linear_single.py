"""GPU tier: the fused LinearProof path (k_lin_single: the host replays each transcript, one thread-block cluster per proof checks its own
equation, one launch).  bp_debug_linear_verify_path forces it (path 1) or the pipeline (path 2) on the same inputs; bp_linear_verify_batch
and bp_linear_verify_mixed route calls of at most ROUTE_COUNT admitted proofs of n <= ROUTE_N to it.  Every verdict must be the oracle's
(orc.linear_verify, with bp.linear_verify beside it) and the pipeline's.  Covered: every k from 0 to LIN_SINGLE_MAX_K, counts 1 to 64,
every damage kind, undecodable and zero points, non-canonical a and r, bad transcript records, transcripts with earlier messages, routed
batch and mixed calls with their launch counts and the non-canonical b refusal, the hook's refusals, a pending range-proof begin, and a
LinearProof reservation and a range-proof reserved geometry that keep verifying after routed calls on the same context."""
import ctypes
import json
import os

import pytest

from oracle_binding import L_ORDER as l
from test_gpu_linear_device import run as device_run
from test_linear_verify_batch import (FORMAT_ERROR, KINDS, OK, VERIFICATION_ERROR, _damaged, _gens, _secret, gpu_proofs, le, lg, single)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_K = 12                              # LIN_SINGLE_MAX_K (linear_single.cuh)
ROUTE_COUNT, ROUTE_N = 16, 1024         # LIN_ROUTE_MAX_COUNT, LIN_ROUTE_MAX_N (linear_single.cuh)
SEED = bytes(range(32))


@pytest.fixture(scope="module")
def bp():
    import bulletproofs_b200
    return bulletproofs_b200


_V = {}


@pytest.fixture(scope="module")
def verifier(bp, gpu_ctx, orc):
    def get(n):
        if n not in _V:
            _V[n] = bp.LinearVerifier(gpu_ctx, *_gens(orc, n))
        return _V[n]
    yield get
    for v in _V.values():
        v.close()
    _V.clear()


def oracle(bp, ctx, orc, n, items):
    gfb = _gens(orc, n)
    return [single(bp, ctx, orc, gfb, p) for p in items]


def both_paths(bp, ctx, V, items, seed=SEED):
    """(fused verdicts, pipeline verdicts, launches of the fused call)"""
    its = [p.item(bp) for p in items]
    l0 = ctx.launches
    fused = ctx.debug_linear_verify_path(V.points, V.n, its, 1, seed)
    nl = ctx.launches - l0
    return fused, ctx.debug_linear_verify_path(V.points, V.n, its, 2, seed), nl


class Record:
    """an item transcript whose 203-byte record is given as it is"""

    def __init__(self, raw):
        self.raw = raw

    def to_bytes(self):
        return self.raw


def edit(p, off, data):
    pr = bytearray(p.proof); pr[off:off + len(data)] = data
    return p.replace(proof=bytes(pr))


def damaged_set(bp, p, n, G):
    """every damage kind of test_linear_verify_batch where n has it, and zero L / R, undecodable C / S / L; G: at least 3 valid points"""
    k = lg(n)
    out = [_damaged(p, kind, n, G) for kind in KINDS if (k >= 1 or kind not in ("L", "R")) and (n > 5 or kind != "b_i")]
    if k >= 1:
        out += [edit(p, 0, bytes(32)), edit(p, 64 * (k - 1) + 32, bytes(32)), edit(p, 0, b"\xff" * 32)]
    out += [p.replace(C=b"\xff" * 32), edit(p, 64 * k, b"\xff" * 32)]
    return out


@pytest.mark.parametrize("k", range(MAX_K + 1))
def test_every_k_fused_equals_pipeline_and_oracle(bp, gpu_ctx, orc, verifier, k):
    n = 1 << k
    V = verifier(n)
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 3)
    items = [proofs[0], _damaged(proofs[1], "a flipped", n, gfb[0]), proofs[2]]
    want = oracle(bp, gpu_ctx, orc, n, items)
    assert want == [OK, VERIFICATION_ERROR, OK]
    fused, pipe, nl = both_paths(bp, gpu_ctx, V, items)
    assert fused == pipe == want and nl == 1
    # the public call of one proof: routed up to ROUTE_N
    l0 = gpu_ctx.launches
    assert V.verify_batch([proofs[0].item(bp)], seed=SEED) == [OK]
    assert (gpu_ctx.launches - l0 == 1) == (n <= ROUTE_N)


@pytest.mark.parametrize("n", [1, 2, 16, 256])
def test_every_damage_kind(bp, gpu_ctx, orc, verifier, n):
    V = verifier(n)
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 1)
    items = [proofs[0]] + damaged_set(bp, proofs[0], n, _gens(orc, 4)[0])
    want = oracle(bp, gpu_ctx, orc, n, items)
    assert want[0] == OK and all(w != OK for w in want[1:]), want
    assert FORMAT_ERROR in want and VERIFICATION_ERROR in want
    for lo in range(0, len(items), 64):
        fused, pipe, nl = both_paths(bp, gpu_ctx, V, items[lo:lo + 64])
        assert fused == pipe == want[lo:lo + 64] and nl == 1


def test_bad_transcript_records(bp, gpu_ctx, orc, verifier):
    """pos at or past the STROBE rate, or pos_begin above pos: FormatError before any replay, on both paths"""
    n = 16
    V = verifier(n)
    proofs, _ = gpu_proofs(bp, gpu_ctx, orc, n, 4)
    its = [p.item(bp) for p in proofs]
    for j, (pos, begin) in enumerate([(166, 0), (255, 3), (10, 11)]):
        raw = bytearray(its[j][0].to_bytes()); raw[200], raw[201] = pos, begin
        its[j] = (Record(bytes(raw)),) + its[j][1:]
    want = [FORMAT_ERROR] * 3 + [OK]
    assert gpu_ctx.debug_linear_verify_path(V.points, n, its, 1) == gpu_ctx.debug_linear_verify_path(V.points, n, its, 2) == want
    assert bp.linear_verify_batch(gpu_ctx, V.points, n, its) == want


def test_transcript_with_earlier_messages(bp, gpu_ctx, orc, verifier):
    n = 64
    V = verifier(n)
    G, F, B = _gens(orc, n)
    a, b, r = _secret(n, 4242)
    rc, C = gpu_ctx.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % l), G + B + F)
    assert rc == 0

    def t():
        x = bp.Transcript(b"linear single"); x.append_message(b"tx", b"hash of the transaction"); return x
    rc, proof = bp.linear_create(gpu_ctx, t(), le(9), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), G, F, B)
    assert rc == 0
    bb = b"".join(map(le, b))
    ot = orc.transcript_append(orc.transcript(b"linear single"), b"tx", b"hash of the transaction")
    assert orc.linear_verify(ot, proof, C, G, F, B, bb) == OK
    good, fresh = (t(), proof, C, bb), (bp.Transcript(b"linear single"), proof, C, bb)
    for path in (1, 2):
        assert gpu_ctx.debug_linear_verify_path(V.points, n, [good, fresh], path) == [OK, VERIFICATION_ERROR]
    assert V.verify_batch([good]) == [OK] and V.verify_batch([fresh]) == [VERIFICATION_ERROR]


@pytest.mark.parametrize("count", [1, 2, 5, 16, 17, 33, 64])
def test_counts_with_one_bad_proof_in_each_slot(bp, gpu_ctx, orc, verifier, count):
    n = 16
    V = verifier(n)
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, count)
    slots = sorted({0, count // 2, count - 1})
    for q in slots:
        items = list(proofs); items[q] = _damaged(items[q], "r flipped", n, gfb[0])
        want = [OK] * count; want[q] = VERIFICATION_ERROR
        fused, pipe, nl = both_paths(bp, gpu_ctx, V, items, seed=bytes([q]) * 32)
        assert fused == pipe == want and nl == 1
        l0 = gpu_ctx.launches
        assert V.verify_batch([p.item(bp) for p in items], seed=SEED) == want
        assert (gpu_ctx.launches - l0 == 1) == (count <= ROUTE_COUNT)


def test_routed_mixed_calls(bp, gpu_ctx, orc, verifier):
    """bp_linear_verify_mixed of at most ROUTE_COUNT admitted proofs up to ROUTE_N: one launch, the oracle's verdicts, parameter codes kept"""
    V = verifier(1024)
    ns = [1, 4, 64, 1024, 16, 256]
    pools = {n: gpu_proofs(bp, gpu_ctx, orc, n, 2) for n in ns}
    items, want = [], []
    for j, n in enumerate(ns):
        p0, p1 = pools[n][0]
        bad = _damaged(p1, "a flipped" if j % 2 else "r flipped", n, pools[n][1][0])
        items += [p0, bad]; want += [OK, VERIFICATION_ERROR]
    short = pools[64][0][0].replace(proof=pools[64][0][0].proof[:-32])          # a length no proof can have: FormatError
    wrong_n = pools[16][0][0].replace(b=pools[16][0][0].b + bytes(32 * 16))   # n = 32 for a proof of 4 rounds: VerificationError
    items += [short, wrong_n]; want += [FORMAT_ERROR, VERIFICATION_ERROR]
    for j, p in enumerate(items[:12]):
        n = len(p.b) // 32
        assert oracle(bp, gpu_ctx, orc, n, [p]) == [want[j]]
    l0 = gpu_ctx.launches
    assert V.verify_mixed([p.item(bp) for p in items], seed=SEED) == want
    assert gpu_ctx.launches - l0 == 1
    # past the rule: ROUTE_COUNT + 1 admitted proofs, or one longer than ROUTE_N, take the pipeline with the same verdicts
    many = [pools[4][0][0]] * (ROUTE_COUNT + 1)
    l0 = gpu_ctx.launches
    assert V.verify_mixed([p.item(bp) for p in many], seed=SEED) == [OK] * (ROUTE_COUNT + 1)
    assert gpu_ctx.launches - l0 > 1
    big = bp.LinearVerifier(gpu_ctx, *_gens(orc, 2048))
    p2k = gpu_proofs(bp, gpu_ctx, orc, 2048, 1)[0][0]
    l0 = gpu_ctx.launches
    assert big.verify_mixed([p.item(bp) for p in (p2k, pools[4][0][0])], seed=SEED) == [OK, OK]
    assert gpu_ctx.launches - l0 > 1
    big.close()


def test_non_canonical_b_refused_on_routed_calls(bp, gpu_ctx, orc, verifier):
    n = 16
    V = verifier(n)
    proofs, _ = gpu_proofs(bp, gpu_ctx, orc, n, 2)
    b = bytearray(proofs[1].b); b[32 * 3:32 * 4] = le(l + 1)
    items = [proofs[0].item(bp), proofs[1].replace(b=bytes(b)).item(bp)]
    for call in (lambda: V.verify_batch(items), lambda: V.verify_mixed(items),
                 lambda: gpu_ctx.debug_linear_verify_path(V.points, n, items, 1), lambda: gpu_ctx.debug_linear_verify_path(V.points, n, items, 2)):
        with pytest.raises(bp.BpError) as e:
            call()
        assert e.value.code == bp.ERR_NONCANONICAL_SCALAR
    assert V.verify_batch(items[:1]) == [OK]


def test_hook_refusals(bp, gpu_ctx, orc, verifier):
    n = 16
    V = verifier(n)
    proofs, _ = gpu_proofs(bp, gpu_ctx, orc, n, 65)
    items = [p.item(bp) for p in proofs]
    for path in (0, 3, -1):
        with pytest.raises(bp.BpError) as e:
            gpu_ctx.debug_linear_verify_path(V.points, n, items[:1], path)
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    with pytest.raises(bp.BpError):
        gpu_ctx.debug_linear_verify_path(V.points, n, items, 1)                  # 65 proofs
    assert gpu_ctx.debug_linear_verify_path(V.points, n, items, 2) == [OK] * 65
    big = bp.LinearVerifier(gpu_ctx, *_gens(orc, 1 << (MAX_K + 1)))
    p = gpu_proofs(bp, gpu_ctx, orc, 1 << (MAX_K + 1), 1)[0][0]
    with pytest.raises(bp.BpError):
        gpu_ctx.debug_linear_verify_path(big.points, big.n, [p.item(bp)], 1)      # k = MAX_K + 1
    assert gpu_ctx.debug_linear_verify_path(big.points, big.n, [p.item(bp)], 2) == [OK]
    big.close()


def test_pending_range_proof_begin_refuses_routed_calls(bp, gpu_ctx, orc, verifier):
    n = 16
    V = verifier(n)
    proofs, _ = gpu_proofs(bp, gpu_ctx, orc, n, 1)
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(gpu_ctx, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)
    bv = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1, reserve=False)
    bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
    for call in (lambda: V.verify_batch([proofs[0].item(bp)]), lambda: V.verify_mixed([proofs[0].item(bp)]),
                 lambda: gpu_ctx.debug_linear_verify_path(V.points, n, [proofs[0].item(bp)], 1)):
        with pytest.raises(bp.BpError) as e:
            call()
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    assert list(bv.finish()) == [OK]
    assert V.verify_batch([proofs[0].item(bp)]) == [OK]
    gens.close()


def test_reserved_graphs_keep_verifying_after_routed_calls(bp, orc):
    """a LinearProof reservation and a range-proof reserved geometry on the context replay with the same verdicts and launch cost after
    routed calls (which never touch their buffers)"""
    c = bp.Context(0)
    try:
        n = 16
        proofs, gfb = gpu_proofs(bp, c, orc, n, 16)
        R = bp.LinearVerifier(c, *gfb, capacity=16)
        reserved_items = proofs[:9] + [_damaged(proofs[9], "R", n, gfb[0])] + proofs[10:]
        first = device_run(bp, R, reserved_items, bytes([1]) * 32)
        assert first[0] == [OK] * 9 + [VERIFICATION_ERROR] + [OK] * 6
        golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
        gens = bp.Gens(c, 64, 1)
        rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
        vc = bytes.fromhex(golden["value_commitments"][0])
        bv = bp.BatchVerifier(c, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1)
        pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)

        def range_call():
            l0 = c.launches
            bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
            assert list(bv.finish()) == [OK]
            return c.launches - l0

        r0 = range_call()
        M = bp.LinearVerifier(c, *_gens(orc, 1024))
        for n2 in (4, 64, 1024):
            ps = gpu_proofs(bp, c, orc, n2, 8)[0]
            bad = list(ps); bad[3] = _damaged(bad[3], "a flipped", n2, None)
            assert bp.linear_verify_batch(c, M.points, n2, [p.item(bp) for p in bad], SEED) == [OK] * 3 + [VERIFICATION_ERROR] + [OK] * 4
            assert M.verify_mixed([p.item(bp) for p in bad], seed=SEED) == [OK] * 3 + [VERIFICATION_ERROR] + [OK] * 4
            assert device_run(bp, R, reserved_items, bytes([1]) * 32) == first
            assert range_call() == r0
        M.close(); gens.close(); R.close()
    finally:
        c.close()
