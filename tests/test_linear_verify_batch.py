"""LinearProof batch verification: bp_linear_verify_batch (transcripts replayed on the device, the generator scalars summed over the proofs,
one combined MSM, each proof's own equation when that MSM does not vanish) through bp.LinearVerifier.  The expected verdict of every
proof is what the single path (bp.linear_verify) and the oracle (orc.linear_verify) return for it.

CPU tier: linear.cuh compiled for the host (tests/host_emul/emul_linear.cpp): the replayed challenges against bp.Transcript, the batching
weight against a Python STROBE, and the tables, b0, the G sums and every MSM scalar against Python integers, for n in {1, 2, 4, 8, 16,
1024}.
GPU tier: valid batches of every size class, single and many bad proofs, points that are the identity or do not decode, parameter
errors, seeds, and n = 4096."""
import ctypes
import os
import random

import pytest

from oracle_binding import L_ORDER as l

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, VERIFICATION_ERROR, FORMAT_ERROR, INVALID_GENERATORS_LENGTH = 0, 1, 2, 4


def le(x, n=32):
    return x.to_bytes(n, "little")


def lg(n):
    return n.bit_length() - 1


# ---------------------------------------------------------------------------------------------------------------------- Python STROBE
# An independent Keccak-f[1600] / STROBE-128 (merlin's framing) for the batching weight:
# build_rng().rekey_with_witness_bytes(label, a || r).finalize(seed) + fill_bytes(64)
_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M = (1 << 64) - 1


def _rol(v, r):
    return ((v << r) | (v >> (64 - r))) & _M if r else v


def _keccak(st: bytearray):
    A = [int.from_bytes(st[8 * i:8 * i + 8], "little") for i in range(25)]
    for rc in _RC:
        C = [A[x] ^ A[x + 5] ^ A[x + 10] ^ A[x + 15] ^ A[x + 20] for x in range(5)]
        A = [A[i] ^ C[(i % 5 - 1) % 5] ^ _rol(C[(i % 5 + 1) % 5], 1) for i in range(25)]
        B = [0] * 25
        for x in range(5):
            for y in range(5):
                B[y + 5 * ((2 * x + 3 * y) % 5)] = _rol(A[x + 5 * y], _ROT[x][y])
        A = [B[i] ^ ((~B[(i + 1) % 5 + 5 * (i // 5)]) & B[(i + 2) % 5 + 5 * (i // 5)]) for i in range(25)]
        A[0] ^= rc
    st[:] = b"".join(le(a, 8) for a in A)


class _Strobe:
    R = 166

    def __init__(self, wire: bytes):
        self.st, self.pos, self.begin = bytearray(wire[:200]), wire[200], wire[201]

    def _run_f(self):
        self.st[self.pos] ^= self.begin; self.st[self.pos + 1] ^= 0x04; self.st[self.R + 1] ^= 0x80
        _keccak(self.st); self.pos = self.begin = 0

    def _step(self):
        self.pos += 1
        if self.pos == self.R:
            self._run_f()

    def absorb(self, d):
        for x in d:
            self.st[self.pos] ^= x; self._step()

    def overwrite(self, d):
        for x in d:
            self.st[self.pos] = x; self._step()

    def squeeze(self, n):
        out = bytearray()
        for _ in range(n):
            out.append(self.st[self.pos]); self.st[self.pos] = 0; self._step()
        return bytes(out)

    def begin_op(self, flags):
        hdr = bytes([self.begin, flags]); self.begin = self.pos + 1
        self.absorb(hdr)
        if flags & (4 | 32) and self.pos != 0:
            self._run_f()


def rng_bytes(wire: bytes, seed: bytes, n: int, label: bytes = None, witness: bytes = None) -> bytes:
    """build_rng(), then rekey_with_witness_bytes(label, witness) when a witness is given, finalize(seed), fill_bytes(n)"""
    s = _Strobe(wire)
    if witness is not None:
        s.begin_op(0x12); s.absorb(label); s.absorb(le(len(witness), 4))
        s.begin_op(0x06); s.overwrite(witness)
    s.begin_op(0x12); s.absorb(b"rng")
    s.begin_op(0x06); s.overwrite(seed)
    s.begin_op(0x12); s.absorb(le(n, 4))
    s.begin_op(0x07); return s.squeeze(n)


# ---------------------------------------------------------------------------------------------------------------------- instances
def _gens(orc, n):
    g = orc.gens(max(n, 1), 1)
    F, B = orc.pedersen()                                           # F = pc_gens.B, B = pc_gens.B_blinding (linear_proof.rs:422-424)
    return b"".join(orc.gens_get(g, 0, 0, i) for i in range(n)), F, B


def _secret(n, seed):
    rnd = random.Random(seed)
    a = [rnd.randrange(l) for _ in range(n)]; b = [rnd.randrange(l) for _ in range(n)]; r = rnd.randrange(l)
    return a, b, r


class Proof:
    """one proof to verify: label, proof bytes, C, b"""

    def __init__(self, label, proof, C, b):
        self.label, self.proof, self.C, self.b = label, proof, C, b

    def replace(self, **kw):
        p = Proof(self.label, self.proof, self.C, self.b)
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    def item(self, bp):
        return (bp.Transcript(self.label), self.proof, self.C, self.b)


def orc_proof(orc, G, F, B, n, seed, label):
    a, b, r = _secret(n, seed)
    rc, C = orc.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % l), G + B + F)
    assert rc == 0
    rc, _, proof = orc.linear_create(orc.transcript(label), le(seed % 2**64, 32), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), G, F, B)
    assert rc == 0
    return Proof(label, proof, C, b"".join(map(le, b)))


_POOL = {}


def gpu_proofs(bp, ctx, orc, n, count, tag="v"):
    """`count` valid proofs at n, proof j under its own label (made with bp.linear_create; cached)"""
    key = (n, tag)
    G, F, B = _gens(orc, n)
    pool = _POOL.setdefault(key, [])
    while len(pool) < count:
        j = len(pool)
        a, b, r = _secret(n, 7919 * n + j)
        rc, C = ctx.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % l), G + B + F)
        assert rc == 0
        label = b"linear batch %s %d %d" % (tag.encode(), n, j)
        rc, proof = bp.linear_create(ctx, bp.Transcript(label), le(j + 1), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), G, F, B)
        assert rc == 0
        pool.append(Proof(label, proof, C, b"".join(map(le, b))))
    return pool[:count], (G, F, B)


def single(bp, ctx, orc, gfb, p):
    G, F, B = gfb
    got = bp.linear_verify(ctx, bp.Transcript(p.label), p.proof, p.C, G, F, B, p.b)
    want = orc.linear_verify(orc.transcript(p.label), p.proof, p.C, G, F, B, p.b)
    assert got == want, (got, want)
    return want


# ---------------------------------------------------------------------------------------------------------------------- CPU tier
@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_lin_transcript.restype = ctypes.c_uint32
    E.emul_recheck_slice.argtypes = [ctypes.c_uint32] * 3; E.emul_recheck_slice.restype = ctypes.c_uint32
    return E


def lin_slice(E, np_, row):
    """proofs per slice of the LinearProof reject path: the shared slice rule with `row` MSM terms per proof and a budget of 2^20"""
    return E.emul_recheck_slice(np_, row, 1 << 20)


def _replay_python(bp, p, n, G, F, B):
    """the verifier's appends made through bp.Transcript (linear_proof.rs:184-197, 272-283): x_j.., x_star and the state after x_star"""
    k = lg(n)
    t = bp.Transcript(p.label)
    t.append_message(b"dom-sep", b"ipp v1"); t.append_u64(b"n", n); t.append_message(b"C", p.C)
    for i in range(n):
        t.append_message(b"b_i", p.b[32 * i:32 * i + 32])
    for i in range(n):
        t.append_message(b"G_i", G[32 * i:32 * i + 32])
    t.append_message(b"F", F); t.append_message(b"B", B)
    xs = []
    for j in range(k):
        t.append_message(b"L", p.proof[64 * j:64 * j + 32]); t.append_message(b"R", p.proof[64 * j + 32:64 * j + 64])
        xs.append(t.challenge_bytes(b"x_j", 64))
    t.append_message(b"S", p.proof[64 * k:64 * k + 32])
    xs.append(t.challenge_bytes(b"x_star", 64))
    return xs, t.to_bytes()


@pytest.mark.parametrize("n", [1, 2, 4, 8, 16, 1024])
def test_replay_rekeyed_weight_and_scalars_against_python(E, orc, n):
    """the weight rho is build_rng().rekey_with_witness_bytes("linear_a_r", a || r).finalize(seed).fill_bytes(64): it depends on
    the proof's a and r, which the transcript never absorbs"""
    import bulletproofs_b200 as bp
    k = lg(n); G, F, B = _gens(orc, n); enc = B + F + G
    proofs = [orc_proof(orc, G, F, B, n, 50 + j, b"emul linear %d %d" % (n, j)) for j in range(3 if n < 1024 else 2)]
    seed = bytes(range(32))
    raws = b""
    for p in proofs:
        raw = ctypes.create_string_buffer(64 * (k + 2))
        assert E.emul_lin_transcript(p.proof, k, n, p.C, p.b, enc, bp.Transcript(p.label).to_bytes(), seed, raw) == OK
        xs, wire = _replay_python(bp, p, n, G, F, B)
        assert [raw.raw[64 * j:64 * j + 64] for j in range(k + 1)] == xs
        assert raw.raw[64 * (k + 1):] == rng_bytes(wire, seed, 64, b"linear_a_r", p.proof[64 * k + 32:64 * k + 96])
        raws += raw.raw
    count, D = len(proofs), 2 + 2 * k
    per = n + 3 + D
    for weighted, chunk in ((1, 2), (0, 1), (1, 32)):
        nch = (count + chunk - 1) // chunk
        out_g, out_p, st = ctypes.create_string_buffer(32 * nch * n), ctypes.create_string_buffer(32 * count * per), (ctypes.c_uint32 * count)()
        plen = len(proofs[0].proof)
        E.emul_lin_scalars(count, k, raws, b"".join(p.proof for p in proofs), plen, b"".join(p.b for p in proofs), weighted, chunk, out_g, out_p, st)
        assert list(st) == [OK] * count
        rd = lambda buf, e: int.from_bytes(buf.raw[32 * e:32 * e + 32], "little")
        want_g = [[0] * n for _ in range(nch)]
        for q, p in enumerate(proofs):
            rw = raws[64 * (k + 2) * q:64 * (k + 2) * (q + 1)]
            x = [int.from_bytes(rw[64 * j:64 * j + 64], "little") % l for j in range(k)]
            xs = int.from_bytes(rw[64 * k:64 * k + 64], "little") % l
            rho = int.from_bytes(rw[64 * (k + 1):], "little") % l if weighted else 1
            a, r = int.from_bytes(p.proof[64 * k + 32:64 * k + 64], "little"), int.from_bytes(p.proof[64 * k + 64:64 * k + 96], "little")
            s = []
            for i in range(n):
                v = 1
                for bit in range(k):
                    if i >> bit & 1:
                        v = v * x[k - 1 - bit] % l
                s.append(v)
            bv = [int.from_bytes(p.b[32 * i:32 * i + 32], "little") for i in range(n)]
            b0 = sum(u * v for u, v in zip(bv, s)) % l
            # the fold of verification_scalars (linear_proof.rs:243-250) gives the same b0
            fold = bv[:]
            for j in range(k):
                h = len(fold) // 2; fold = [(fold[i] + x[j] * fold[h + i]) % l for i in range(h)]
            assert fold == [b0]
            base = q * per
            assert [rd(out_p, base + i) for i in range(n)] == s
            assert [rd(out_p, base + n + e) for e in range(3)] == [b0, rho * r % l, rho * a * b0 % l]
            dyn = [-rho * xs, -rho] + [-rho * xs * xj for xj in x] + [-rho * xs * pow(xj, l - 2, l) for xj in x]
            assert [rd(out_p, base + n + 3 + d) for d in range(D)] == [v % l for v in dyn]
            for i in range(n):
                want_g[q // chunk][i] = (want_g[q // chunk][i] + rho * a * s[i]) % l
        assert [[rd(out_g, c * n + i) for i in range(n)] for c in range(nch)] == want_g
        if not weighted:                                            # each proof's own equation, through the oracle's MSM: the identity
            for q, p in enumerate(proofs):
                sc = b"".join(le(rd(out_p, q * per + n + e)) for e in (1, 2)) + out_g.raw[32 * q * n:32 * (q + 1) * n] + out_p.raw[32 * (q * per + n + 3):32 * (q + 1) * per]
                k_ = k; pr = p.proof
                pts = B + F + G + p.C + pr[64 * k_:64 * k_ + 32] + b"".join(pr[64 * j:64 * j + 32] for j in range(k_)) + b"".join(pr[64 * j + 32:64 * j + 64] for j in range(k_))
                assert orc.msm(sc, pts) == (0, bytes(32))


def test_replay_rejects_identity_points_and_non_canonical_scalars(E, orc):
    import bulletproofs_b200 as bp
    n, k = 16, 4; G, F, B = _gens(orc, n)
    p = orc_proof(orc, G, F, B, n, 3, b"emul linear edge")
    raw = ctypes.create_string_buffer(64 * (k + 2))
    run = lambda proof: E.emul_lin_transcript(proof, k, n, p.C, p.b, B + F + G, bp.Transcript(p.label).to_bytes(), bytes(32), raw)
    pr = bytearray(p.proof); pr[64:96] = bytes(32)                 # L_1 = identity
    assert run(bytes(pr)) == VERIFICATION_ERROR
    pr = bytearray(p.proof); pr[64 * 3 + 32:64 * 3 + 64] = bytes(32)                 # R_3 = identity
    assert run(bytes(pr)) == VERIFICATION_ERROR
    for off in (64 * k + 32, 64 * k + 64):                          # a, r >= l
        pr = bytearray(p.proof); pr[off:off + 32] = le(l)
        assert run(bytes(pr)) == FORMAT_ERROR
    assert run(p.proof) == OK


def test_reject_path_slice_rule(E):
    f = lambda np_, row: lin_slice(E, np_, row)
    assert (f(1030, 1024 + 2 + 22), f(5, 1048), f(70000, 16), f(3, 1 << 21)) == (1000, 5, 65535, 1)
    for np_ in (1, 999, 1000, 1001, 70000):
        for row in (4, 100, 1048, 4122, 1 << 20, 1 << 21):
            assert f(np_, row) == min(np_, 65535, max(1, (1 << 20) // row))


# ---------------------------------------------------------------------------------------------------------------------- GPU tier
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 16, 64, 1024])
def test_valid_batches_every_size_class(gpu_ctx, orc, n):
    import bulletproofs_b200 as bp
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 257)
    want = [single(bp, gpu_ctx, orc, gfb, p) for p in proofs]
    assert want == [OK] * 257
    V = bp.LinearVerifier(gpu_ctx, *gfb)
    for count in (1, 2, 31, 32, 33, 257):
        assert V.verify_batch([p.item(bp) for p in proofs[:count]], seed=bytes([count % 256]) * 32) == [OK] * count, count
    V.close()


def _damaged(p, kind, n, G):
    k = lg(n); pr = bytearray(p.proof)
    if kind == "L":
        pr[0:32] = G[0:32]                                          # another valid point
    elif kind == "R":
        pr[64 * (k - 1) + 32] ^= 1                                  # last R, one bit
    elif kind == "S":
        pr[64 * k:64 * k + 32] = G[32:64]
    elif kind == "a flipped":
        pr[64 * k + 32] ^= 1
    elif kind == "a non-canonical":
        pr[64 * k + 32:64 * k + 64] = le(l)
    elif kind == "r flipped":
        pr[64 * k + 64] ^= 1
    elif kind == "r non-canonical":
        pr[64 * k + 64:64 * k + 96] = le(l + 5)
    elif kind == "C":
        return p.replace(C=G[64:96])
    elif kind == "b_i":
        b = bytearray(p.b); b[32 * 5] ^= 2; return p.replace(b=bytes(b))
    elif kind == "label":
        return p.replace(label=p.label + b"!")
    return p.replace(proof=bytes(pr))


KINDS = ["L", "R", "S", "a flipped", "a non-canonical", "r flipped", "r non-canonical", "C", "b_i", "label"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_one_bad_proof_among_64(gpu_ctx, orc, kind):
    import bulletproofs_b200 as bp
    n = 16
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 64)
    bad = _damaged(proofs[17], kind, n, gfb[0])
    code = single(bp, gpu_ctx, orc, gfb, bad)
    assert code == (FORMAT_ERROR if "non-canonical" in kind else VERIFICATION_ERROR)
    items = proofs[:17] + [bad] + proofs[18:]
    V = bp.LinearVerifier(gpu_ctx, *gfb)
    assert V.verify_batch([p.item(bp) for p in items], seed=bytes(32)) == [OK] * 17 + [code] + [OK] * 46
    V.close()


@pytest.mark.gpu
def test_every_proof_bad(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n = 64
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 40)
    items = [_damaged(p, KINDS[j % len(KINDS)], n, gfb[0]) for j, p in enumerate(proofs)]
    want = [single(bp, gpu_ctx, orc, gfb, p) for p in items]
    assert OK not in want
    V = bp.LinearVerifier(gpu_ctx, *gfb)
    assert V.verify_batch([p.item(bp) for p in items]) == want
    V.close()


@pytest.mark.gpu
def test_more_bad_proofs_than_one_reject_slice(gpu_ctx, orc, E):
    """1030 proofs at n = 1024: the reject path re-checks them in two slices, [0, 1000) and [1000, 1030), with bad proofs in both"""
    import bulletproofs_b200 as bp
    n, count = 1024, 1030
    per = lin_slice(E, count, n + 2 + 2 + 2 * lg(n))
    assert per == 1000, "the slice rule moved: update the layout of this test"
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 4)
    bads = [_damaged(proofs[j], kind, n, gfb[0]) for j, kind in enumerate(("a flipped", "R", "C", "b_i"))]
    want_bad = [single(bp, gpu_ctx, orc, gfb, p) for p in bads]
    bad_at = set(range(0, count, 3)) | {999, 1000, 1029}
    items = [bads[i % 4] if i in bad_at else proofs[i % 4] for i in range(count)]
    want = [want_bad[i % 4] if i in bad_at else OK for i in range(count)]
    V = bp.LinearVerifier(gpu_ctx, *gfb)
    got = V.verify_batch([p.item(bp) for p in items], seed=bytes(range(32)))
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:10]
    V.close()


@pytest.mark.gpu
def test_identity_and_undecodable_points(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n = 16; k = lg(n)
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 32)
    V = bp.LinearVerifier(gpu_ctx, *gfb)

    def edit(p, off, data):
        pr = bytearray(p.proof); pr[off:off + 32] = data; return p.replace(proof=bytes(pr))

    zero_L, zero_R = edit(proofs[3], 64, bytes(32)), edit(proofs[4], 64 * 2 + 32, bytes(32))
    undec_C, undec_S = proofs[5].replace(C=b"\xff" * 32), edit(proofs[6], 64 * k, b"\xff" * 32)
    for p in (zero_L, zero_R, undec_C, undec_S):
        assert single(bp, gpu_ctx, orc, gfb, p) == VERIFICATION_ERROR

    def launches(items):
        n0 = gpu_ctx.launches
        got = V.verify_batch([p.item(bp) for p in items], seed=bytes(32))
        return got, gpu_ctx.launches - n0

    got, ok_launches = launches(proofs)
    assert got == [OK] * 32
    items = proofs[:3] + [zero_L, zero_R, undec_C, undec_S] + proofs[7:]
    got, nl = launches(items)
    assert got == [OK] * 3 + [VERIFICATION_ERROR] * 4 + [OK] * 25
    undecodable = proofs[:5] + [undec_C, undec_S] + proofs[7:]     # decided by the combined check alone
    got, nl = launches(undecodable)
    assert got == [OK] * 5 + [VERIFICATION_ERROR] * 2 + [OK] * 25 and nl == ok_launches
    got, nl = launches(proofs[:9] + [_damaged(proofs[9], "a flipped", n, gfb[0])] + proofs[10:])
    assert got == [OK] * 9 + [VERIFICATION_ERROR] + [OK] * 22 and nl > ok_launches
    V.close()


@pytest.mark.gpu
def test_parameters(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n = 16
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 5)
    G, F, B = gfb
    V = bp.LinearVerifier(gpu_ctx, G, F, B)
    # a length no proof can have: FormatError for every proof, as LinearProof::from_bytes
    trunc = [p.replace(proof=p.proof[:-32]) for p in proofs]
    assert single(bp, gpu_ctx, orc, gfb, trunc[0]) == FORMAT_ERROR
    assert V.verify_batch([p.item(bp) for p in trunc]) == [FORMAT_ERROR] * 5
    # a well-formed length of 3 rounds against n = 16: VerificationError, and FormatError for a proof with a non-canonical a
    short8, gfb8 = gpu_proofs(bp, gpu_ctx, orc, 8, 3)
    items = [p.replace(b=proofs[0].b) for p in short8]
    items[1] = _damaged(items[1], "a non-canonical", 8, G)
    want = [single(bp, gpu_ctx, orc, gfb, p) for p in items]
    assert want == [VERIFICATION_ERROR, FORMAT_ERROR, VERIFICATION_ERROR]
    assert V.verify_batch([p.item(bp) for p in items]) == want
    # a set with fewer than n + 2 points: InvalidGeneratorsLength
    small = bp.PointSet(gpu_ctx, B + F + G[:32 * (n - 1)])
    assert bp.linear_verify_batch(gpu_ctx, small, n, [p.item(bp) for p in proofs]) == [INVALID_GENERATORS_LENGTH] * 5
    small.close()
    # a b entry >= l is a caller error
    bad_b = bytearray(proofs[2].b); bad_b[32 * 3:32 * 4] = le(l)
    with pytest.raises(bp.BpError) as e:
        V.verify_batch([p.item(bp) for p in proofs[:2]] + [proofs[2].replace(b=bytes(bad_b)).item(bp)])
    assert e.value.code == bp.ERR_NONCANONICAL_SCALAR
    # NULL or empty arguments
    L = bp.lib(); vd = ctypes.create_string_buffer(5); p0 = proofs[0]
    args = lambda **kw: dict(dict(set=V.points._h, count=1, t=bp.Transcript(p0.label).to_bytes(), proofs=p0.proof, C=p0.C, b=p0.b), **kw)
    for kw in (dict(count=0), dict(proofs=None), dict(t=None), dict(C=None), dict(b=None), dict(set=None)):
        a = args(**kw)
        assert L.bp_linear_verify_batch(gpu_ctx._h, a["set"], n, a["count"], a["t"], a["proofs"], len(p0.proof), a["C"], a["b"], None, vd) == bp.ERR_INVALID_ARGUMENT, kw
    # a pending range-proof verification on the context
    golden = __import__("json").load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(gpu_ctx, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    bv = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1, reserve=False)
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)
    bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
    with pytest.raises(bp.BpError) as e:
        V.verify_batch([p.item(bp) for p in proofs])
    assert e.value.code == bp.ERR_INVALID_ARGUMENT
    assert list(bv.finish()) == [OK]
    assert V.verify_batch([p.item(bp) for p in proofs]) == [OK] * 5
    gens.close(); V.close()


@pytest.mark.gpu
def test_seeds(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n = 64
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 33)
    items = proofs[:20] + [_damaged(proofs[20], "S", n, gfb[0])] + proofs[21:]
    V = bp.LinearVerifier(gpu_ctx, *gfb)
    want = [OK] * 20 + [VERIFICATION_ERROR] + [OK] * 12
    for seed in (bytes(32), bytes([0xA5]) * 32, None):
        assert V.verify_batch([p.item(bp) for p in items], seed=seed) == want
    V.close()


@pytest.mark.gpu
def test_n_4096_agrees_with_the_oracle(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n = 4096
    proofs, gfb = gpu_proofs(bp, gpu_ctx, orc, n, 8)
    items = proofs[:5] + [_damaged(proofs[5], "b_i", n, gfb[0])] + proofs[6:]
    G, F, B = gfb
    want = [orc.linear_verify(orc.transcript(p.label), p.proof, p.C, G, F, B, p.b) for p in items]
    assert want == [OK] * 5 + [VERIFICATION_ERROR] + [OK] * 2
    V = bp.LinearVerifier(gpu_ctx, *gfb)
    assert V.verify_batch([p.item(bp) for p in items]) == want
    V.close()
