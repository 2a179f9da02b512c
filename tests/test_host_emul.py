"""CPU tier: the device math headers (fe/ge/sc/merlin/rp/msm_common .cuh) compiled for the host by
tests/host_emul/emul.cpp, checked against Python big integers and the oracle.  This covers the limb
algorithms' portable branches, every point formula, the transcript replay, the verification-scalar
assembly (on all 16 golden proofs) and the Pippenger bookkeeping.  The PTX branches and the kernels
themselves are covered by the -m gpu tier."""
import ctypes
import os
import random

import pytest

from oracle_binding import L_ORDER as l, P_FIELD as p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def E(built):
    return ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))


def buf(n=32):
    return ctypes.create_string_buffer(n)


def le(x, n=32):
    return x.to_bytes(n, "little")


def test_field_ops(E):
    rnd = random.Random(1)
    edge = [0, 1, 2, p - 1, p, p + 1, 2**255 - 1, 2**255, 2**256 - 1, 2**256 - 38, 2**256 - 39, 38, 19, p + 5]
    vals = edge + [rnd.getrandbits(256) for _ in range(300)]
    fns = ((0, lambda a, b: (a + b) % p), (1, lambda a, b: (a - b) % p), (2, lambda a, b: a * b % p), (5, lambda a, b: (-a) % p), (6, lambda a, b: a * a % p))
    for _ in range(1500):
        a, b = rnd.choice(vals), rnd.choice(vals)
        for op, f in fns:
            o = buf(); E.emul_fe_op(op, le(a), le(b), o)
            assert int.from_bytes(o.raw, "little") == f(a, b), (op, a, b)
    for a in vals[:40]:
        o = buf(); E.emul_fe_op(3, le(a), bytes(32), o); assert int.from_bytes(o.raw, "little") == pow(a % p, p - 2, p)
        o = buf(); E.emul_fe_op(4, le(a), bytes(32), o); assert int.from_bytes(o.raw, "little") == pow(a % p, (p - 5) // 8, p)


def test_scalar_ops(E):
    rnd = random.Random(2)
    for _ in range(400):
        a, b = rnd.randrange(l), rnd.randrange(l)
        o = buf(); E.emul_sc_mul(le(a), le(b), o); assert int.from_bytes(o.raw, "little") == a * b % l
        o = buf(); E.emul_sc_addsub(le(a), le(b), 0, o); assert int.from_bytes(o.raw, "little") == (a + b) % l
        o = buf(); E.emul_sc_addsub(le(a), le(b), 1, o); assert int.from_bytes(o.raw, "little") == (a - b) % l
        w = rnd.getrandbits(512); o = buf(); E.emul_sc_from_wide(le(w, 64), o); assert int.from_bytes(o.raw, "little") == w % l
    for a in [1, 2, l - 1] + [rnd.randrange(1, l) for _ in range(8)]:
        o = buf(); E.emul_sc_invert(le(a), o); assert int.from_bytes(o.raw, "little") == pow(a, l - 2, l)


def test_merlin(E, orc):
    st = buf(203); E.emul_transcript_new(b"test protocol", 13, st); E.emul_transcript_append(st, b"some label", b"some data", 9)
    ch = buf(32); E.emul_transcript_challenge(st, b"challenge", ch, 32)
    assert ch.raw.hex() == "d5a21972d0d5fe320c0d263fac7fffb8145aa640af6e9bca177c03c7efcf0615"
    st3 = buf(203); E.emul_transcript_new(b"abc", 3, st3)
    assert orc.transcript(b"abc")[:203] == st3.raw


def test_lazy_reduction_of_product_sums(E):
    """sc_wide_mac / sc_wide_redc (k_rp_scalars_sum): up to 32 products summed as 512-bit integers, one Montgomery reduction"""
    rnd = random.Random(12)
    for n, mode in [(1, "rand"), (7, "rand"), (32, "rand"), (32, "max"), (32, "zero"), (31, "mixed")]:
        if mode == "max": A = [l - 1] * n; B = [l - 1] * n
        elif mode == "zero": A = [0] * n; B = [rnd.randrange(l) for _ in range(n)]
        elif mode == "mixed": A = [rnd.choice([0, 1, l - 1, rnd.randrange(l)]) for _ in range(n)]; B = [rnd.choice([l - 1, l - 2, rnd.randrange(l)]) for _ in range(n)]
        else: A = [rnd.randrange(l) for _ in range(n)]; B = [rnd.randrange(l) for _ in range(n)]
        o = buf(); E.emul_sc_sum_products(b"".join(le(x) for x in A), b"".join(le(x) for x in B), n, o)
        assert int.from_bytes(o.raw, "little") == sum(x * y for x, y in zip(A, B)) % l, (n, mode)


def test_points(E, orc):
    rnd = random.Random(3)
    pts = []
    for _ in range(120):
        u = rnd.randbytes(64); o = buf(); E.emul_from_uniform(u, o)
        assert o.raw == orc.from_uniform(u)
        pts.append(o.raw)
        o3 = buf(); assert E.emul_point_roundtrip(o.raw, o3) == 1 and o3.raw == o.raw
        o5 = buf(); E.emul_point_double_encode(o.raw, o5); assert o5.raw == orc.point_double_encode(o.raw)
    for _ in range(60):
        a, b = rnd.choice(pts), rnd.choice(pts); o = buf()
        assert E.emul_point_add(a, b, 0, o) == 1 and o.raw == orc.point_add(a, b)
        assert E.emul_point_add(a, b, 1, o) == 1
        assert E.emul_is_identity_of_diff(a, a) == 1 and (a == b or E.emul_is_identity_of_diff(a, b) == 0)
    # malformed encodings: same accept/reject as the oracle
    for i in range(1500):
        s = bytearray(rnd.randbytes(32))
        if i % 4 == 0: s[31] |= 0x80
        if i % 7 == 0:
            s = bytearray(rnd.choice(pts)); s[rnd.randrange(32)] ^= 1 << rnd.randrange(8)
        assert orc.point_is_valid(bytes(s)) == E.emul_point_roundtrip(bytes(s), buf())
    for s in (bytes(32), le(p), le(p + 2), le(1), le(2**255 - 20), b"\xff" * 32):
        assert orc.point_is_valid(s) == E.emul_point_roundtrip(s, buf()), s.hex()


def test_pippenger_bookkeeping(E, orc):
    rnd = random.Random(4)
    pts = [orc.from_uniform(rnd.randbytes(64)) for _ in range(30)]
    for n, c, nt in ((1, 3, 32), (5, 4, 32), (40, 5, 32), (150, 6, 32), (150, 7, 64), (200, 9, 256), (64, 8, 32), (20, 13, 256), (6, 16, 256)):
        sc = b"".join(le(rnd.randrange(l)) for _ in range(n)); pp = b"".join(rnd.choice(pts) for _ in range(n))
        o = buf(); assert E.emul_msm(sc, pp, n, c, nt, o) == 0
        assert (0, o.raw) == orc.msm(sc, pp), (n, c)
    sc = b"".join(le(x) for x in (0, 1, l - 1, 2**252, 2**128, l - 2**200)); pp = b"".join(pts[:6])
    for c in (3, 7, 11, 16):
        o = buf(); E.emul_msm(sc, pp, 6, c, 32, o); assert (0, o.raw) == orc.msm(sc, pp)


def test_window_table(E):
    """msm_pick_window: monotone in the MSM size, every window count covers 253 bits plus the recoding carry, and from 17 terms up
    the width never divides 252 (a width that does leaves a carry-only top window whose single bucket receives half the terms)."""
    import ctypes
    E.emul_pick_window.argtypes = [ctypes.c_uint64]
    prev = 0
    for lg4 in range(0, 4 * 26):
        n = int(2 ** (lg4 / 4))
        c = E.emul_pick_window(n)
        assert 3 <= c <= 16 and c >= prev; prev = c
        assert E.emul_num_windows(c) * c >= 253
        if n > 16: assert 252 % c != 0, (n, c)


def test_pipeline_branch_selection(E):
    """The shared selection rules of msm_common.cuh / rp.cuh that the GPU branch tests rely on: the heavy-bucket threshold sits far
    above the mean bucket size and never below 256, the two-lane accumulate needs >= 8 terms per bucket on average and fewer than
    65536 buckets, combine4 takes up to 256 MSMs, and the verifier re-checks a whole batch once more than four chunks of 32 fail."""
    E.emul_avg_terms.argtypes = [ctypes.c_uint64, ctypes.c_uint32]; E.emul_avg_terms.restype = ctypes.c_uint64
    E.emul_heavy_min.argtypes = [ctypes.c_uint64, ctypes.c_uint32]; E.emul_heavy_min.restype = ctypes.c_uint32
    E.emul_acc_split.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint64]
    E.emul_use_combine4.argtypes = [ctypes.c_uint32]
    E.emul_rp_recheck_whole_batch.argtypes = [ctypes.c_uint32]
    assert [E.emul_avg_terms(T, n) for T, n in ((1, 1), (2000, 1), (2001, 2), (139394, 1), (10, 257))] == [1, 2000, 1001, 139394, 1]
    for avg in (1, 8, 300, 2000, 17538, 139394, 1 << 20):
        for c in range(2, 19):
            nb = 1 << (c - 1); h = E.emul_heavy_min(avg, nb)
            assert h >= 256 and h > 8 * avg / nb, (avg, c, h)
            assert E.emul_heavy_min(avg + nb, nb) >= h
    assert E.emul_heavy_min(300, 16) == 256 and E.emul_heavy_min(2000, 128) == 256 and E.emul_heavy_min(139394, 4096) == 280
    assert E.emul_acc_split(2000, 128, 32 * 128) == 2 and E.emul_acc_split(300, 16, 8 * 51 * 16) == 2
    assert E.emul_acc_split(1023, 128, 32 * 128) == 1 and E.emul_acc_split(300, 16, 300 * 51 * 16) == 1
    assert [E.emul_use_combine4(n) for n in (1, 255, 256, 257, 1024)] == [1, 1, 1, 0, 0]
    assert E.emul_rp_chunk() == 32
    assert [E.emul_rp_recheck_whole_batch(n) for n in (0, 1, 4, 5, 6, 32)] == [0, 0, 0, 1, 1, 1]


def test_bucket_counts_follow_the_recoding(E):
    """emul_bucket_counts (the GPU branch tests' bucket sizes) against the signed-digit recoding written out with Python integers:
    digit_w = window w of (s + sum_w 2^(c w + c - 1)) minus 2^(c-1), and sum_w digit_w 2^(c w) = s"""
    rnd = random.Random(14)
    for c in (3, 5, 8, 13, 17, 18):
        W = E.emul_num_windows(c); nb = 1 << (c - 1)
        vals = [0, 1, l - 1, 2**252] + [rnd.randrange(l) for _ in range(50)]
        want = [0] * (W * nb)
        for s in vals:
            r = s + sum(1 << (c * w + c - 1) for w in range(W))
            digits = [((r >> (c * w)) & ((1 << c) - 1)) - nb for w in range(W)]
            assert sum(d << (c * w) for w, d in enumerate(digits)) == s
            for w, d in enumerate(digits):
                if d: want[w * nb + abs(d) - 1] += 1
        counts = (ctypes.c_uint32 * (W * nb))()
        assert E.emul_bucket_counts(b"".join(le(s) for s in vals), len(vals), c, counts) == 0
        assert list(counts) == want, c


def test_verification_scalars_on_golden_proofs(E, orc, golden):
    """sum scalars * points of the device-side scalar assembly must be the identity for every golden
    proof (RangeProof::verify_multiple accepts) and must not be after a one-bit change."""
    g = orc.gens(64, 8)
    vc = b"".join(bytes.fromhex(v) for v in golden["value_commitments"])
    B, Bb = orc.pedersen()
    lab = golden["transcript_label"].encode(); st = buf(203); E.emul_transcript_new(lab, len(lab), st)
    rnd = random.Random(5)
    for pr in golden["proofs"]:
        n, m = pr["n"], pr["m"]; pb = bytes.fromhex(pr["proof"]); N = n * m; k = N.bit_length() - 1; S = 2 + 2 * N; D = 4 + 2 * k + m
        pts = [Bb, B] + [orc.gens_get(g, w, j, i) for w in (0, 1) for j in range(m) for i in range(n)]
        pts += [pb[0:32], pb[32:64], pb[64:96], pb[96:128]] + [pb[224 + 64 * j:256 + 64 * j] for j in range(k)] + [pb[256 + 64 * j:288 + 64 * j] for j in range(k)] + [vc[32 * j:32 * j + 32] for j in range(m)]
        assert len(pts) == S + D
        for tamper in (0, 1):
            pbb = bytearray(pb)
            if tamper: pbb[200] ^= 4
            out = buf(32 * (S + D))
            assert E.emul_rp_scalars(bytes(pbb), k, vc, n, m, st.raw, rnd.randbytes(32), out) == 0
            rc, res = orc.msm(out.raw, b"".join(pts))
            assert rc == 0 and (res == bytes(32)) == (not tamper), (n, m, tamper)
    # non-canonical scalar in the proof -> FormatError (2); identity point A -> VerificationError (1)
    pb = bytearray(bytes.fromhex(golden["proofs"][0]["proof"])); pb[128:160] = b"\xff" * 32
    assert E.emul_rp_scalars(bytes(pb), 3, vc, 8, 1, st.raw, bytes(32), buf(32 * 30)) == 2
    pb = bytearray(bytes.fromhex(golden["proofs"][0]["proof"])); pb[0:32] = bytes(32)
    assert E.emul_rp_scalars(bytes(pb), 3, vc, 8, 1, st.raw, bytes(32), buf(32 * 30)) == 1


GRID = [(n, m) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32)]      # the reference's range-proof benchmark grid


def test_verification_scalars_on_the_whole_grid(E, orc):
    """The scalar assembly at every (n, m) the reference benchmarks, m up to 32 (N = 2048, S = 4098 static terms, V powers up to
    z^31).  rp_scalars_head splits the k index bits in a low group of kl = ceil(k/2) bits (TL = 2^kl) and a high group; F(i) =
    2^(i mod n) z^(i div n) goes to the low-group table P_lo when TL > n, to the high-group table P_hi when TL <= n.  Per cell: one
    oracle proof must give the identity, and a changed t_x, b, last R or last V must not."""
    E.emul_rp_kl.argtypes = [ctypes.c_uint32]; E.emul_rp_kl.restype = ctypes.c_uint32
    kl = {(n, m): E.emul_rp_kl((n * m).bit_length() - 1) for n, m in GRID}
    above = sorted(c for c in GRID if 1 << kl[c] > c[0])
    assert above == [(8, 16), (8, 32), (16, 32)], f"cells with TL > n: {above}"
    assert any(1 << kl[c] == c[0] for c in GRID) and any(1 << kl[c] < c[0] for c in GRID)
    og = orc.gens(64, 32)
    B, Bb = orc.pedersen()
    label = b"AggregateRangeProofBenchmark"; st = buf(203); E.emul_transcript_new(label, len(label), st)
    rnd = random.Random(24)
    wrong = []
    for n, m in GRID:
        N = n * m; k = N.bit_length() - 1; S = 2 + 2 * N; D = 4 + 2 * k + m
        values = [rnd.randrange(1 << n) for _ in range(m)]
        rc, pb, vc = orc.rangeproof_prove(og, orc.transcript(label), values, b"".join(le(rnd.randrange(l)) for _ in range(m)), n, seed=le(1000 * n + m))
        assert rc == 0 and len(pb) == 32 * (9 + 2 * k)
        static = [Bb, B] + [orc.gens_get(og, w, j, i) for w in (0, 1) for j in range(m) for i in range(n)]
        r_last, v_last = 224 + 64 * (k - 1) + 32, 32 * (m - 1)
        cases = {"valid": (pb, vc),
                 "t_x": (pb[:128] + bytes([pb[128] ^ 1]) + pb[129:], vc),
                 "b": (pb[:-32] + bytes([pb[-32] ^ 1]) + pb[-31:], vc),
                 "last R": (pb[:r_last] + orc.point_double_encode(pb[r_last:r_last + 32]) + pb[r_last + 32:], vc),
                 "last V": (pb, vc[:v_last] + orc.point_double_encode(vc[v_last:]))}
        for name, (p_, v_) in cases.items():
            dyn = [p_[0:32], p_[32:64], p_[64:96], p_[96:128]] + [p_[224 + 64 * j:256 + 64 * j] for j in range(k)] + \
                  [p_[256 + 64 * j:288 + 64 * j] for j in range(k)] + [v_[32 * j:32 * j + 32] for j in range(m)]
            out = buf(32 * (S + D))
            assert E.emul_rp_scalars(p_, k, v_, n, m, st.raw, rnd.randbytes(32), out) == 0, (n, m, name)
            rc, res = orc.msm(out.raw, b"".join(static + dyn))
            assert rc == 0, (n, m, name)
            if (res == bytes(32)) != (name == "valid"):
                wrong.append((n, m, name))
    assert wrong == [], f"(n, m, case) with the wrong outcome: {wrong}"
