"""R1CS batch verification: bp_r1cs_verify_batch (the G/H scalars summed over the proofs on the device, one combined MSM, each proof's
own mega-check when that MSM does not vanish) through r1cs::verify_batch and bp.r1cs_verify_batch.  The expected verdict of every
proof is the oracle's per-proof r1cs_verify.

GPU tier: mixed batches of shuffles, example and range gadgets, valid and damaged in every way the verifier distinguishes; a batch
of one; permuted batches; a gens table too small for one proof; 1024 proofs with one and with many bad ones; 4 x 4096 multipliers;
600 proofs around one of 4096 multipliers, re-checked in two slices.
CPU tier: the device's weighted G/H sums (r1cs.cuh, compiled for the host) against Python integers, the reject path's slice rule, and this file's GPU tests
through the mock engine (tests/mock_engine/mock_r1cs.c: the same C ABI on the oracle's CPU arithmetic, one MSM per proof)."""
import ctypes
import os
import random
import subprocess
import sys

import pytest

from oracle_binding import L_ORDER as l

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# BP_TEST_R1CS_MOCK=1 (set only by test_batch_tests_through_the_mock_engine for its child process): the Python binding and the C++ host
# mirror run against tests/mock_engine/libmockbpmsm_r1cs.so, the mock engine with bp_r1cs_verify_batch (tests/mock_engine/mock_r1cs.c)
if os.environ.get("BP_TEST_R1CS_MOCK") == "1":
    import bulletproofs_b200 as _bp
    _bp.LIB_PATH = os.path.join(ROOT, "tests", "mock_engine", "libmockbpmsm_r1cs.so")
    _bp.HOST_LIB_PATH = os.path.join(ROOT, "tests", "mock_engine", "libbulletproofs_host_mock_r1cs.so")
SHUFFLE, EXAMPLE, RANGE = 0, 1, 2
OK, VERIFICATION_ERROR, FORMAT_ERROR, INVALID_GENERATORS_LENGTH = 0, 1, 2, 4


def le(x, n=32):
    return x.to_bytes(n, "little")


class Item:
    """one proof to verify: the two transcripts (engine binding, oracle), gadget, commitments, proof bytes, param"""

    def __init__(self, name, label, k, gadget, V, proof, param=0):
        self.name, self.label, self.k, self.gadget, self.V, self.proof, self.param = name, label, k, gadget, V, proof, param

    def replace(self, name, **kw):
        it = Item(name, self.label, self.k, self.gadget, self.V, self.proof, self.param)
        for key, v in kw.items():
            setattr(it, key, v)
        return it

    def bp_transcript(self, bp):
        t = bp.Transcript(self.label)
        if self.gadget == SHUFFLE:
            t.append_message(b"dom-sep", b"ShuffleProof"); t.append_u64(b"k", self.k)
        return t

    def orc_transcript(self, orc):
        t = orc.transcript(self.label)
        if self.gadget == SHUFFLE:
            t = orc.transcript_append(t, b"dom-sep", b"ShuffleProof"); t = orc.transcript_append(t, b"k", le(self.k, 8))
        return t

    def batch_item(self, bp):
        return (self.bp_transcript(bp), self.gadget, self.V, self.proof, self.param)

    def expected(self, orc, og):
        return orc.r1cs_verify(og, self.orc_transcript(orc), self.gadget, self.V, self.proof, param=self.param)

    # byte offsets in R1CSProof::to_bytes (proof.rs:83-204)
    def _points(self):
        return 11 if self.proof[0] == 1 else 8

    def off_T1(self):
        return 1 + 32 * (self._points() - 5)

    def off_scalars(self):
        return 1 + 32 * self._points()


_CACHE = {}


def shuffle_item(orc, og, k, seed, permutation=True, name=None):
    key = ("shuffle", k, seed, permutation)
    if key not in _CACHE:
        rnd = random.Random(seed)
        inp = [rnd.randrange(1 << 64) for _ in range(k)]; out = inp[:]; rnd.shuffle(out)
        if not permutation:
            out[-1] ^= 1
        bl = b"".join(le(rnd.randrange(l)) for _ in range(2 * k))
        it = Item(name or f"shuffle{k}", b"ShuffleProofTest", k, SHUFFLE, None, None)
        rc, it.proof, it.V = orc.r1cs_prove(og, it.orc_transcript(orc), SHUFFLE, inp + out, bl)
        assert rc == 0
        _CACHE[key] = it
    return _CACHE[key]


def example_item(orc, og):
    if "example" not in _CACHE:
        rnd = random.Random(9)
        bl = b"".join(le(rnd.randrange(l)) for _ in range(5))
        rc, proof, V = orc.r1cs_prove(og, orc.transcript(b"R1CSExampleGadget"), EXAMPLE, [3, 4, 6, 1, 40], bl, param=9)
        assert rc == 0
        _CACHE["example"] = Item("example", b"R1CSExampleGadget", 0, EXAMPLE, V, proof, param=9)
    return _CACHE["example"]


def range_item(orc, og, n, seed):
    key = ("range", n, seed)
    if key not in _CACHE:
        rnd = random.Random(seed)
        v = rnd.randrange(1 << n)
        rc, proof, V = orc.r1cs_prove(og, orc.transcript(b"RangeProofTest"), RANGE, [v], le(rnd.randrange(l)), param=n, aux=v)
        assert rc == 0
        _CACHE[key] = Item(f"range{n}", b"RangeProofTest", 0, RANGE, V, proof, param=n)
    return _CACHE[key]


def valid_items(orc, og):
    """shuffles with k in {1, 2, 5, 42}, the example gadget (padded_n = 1, no IPP rounds) and range gadgets with n = 10 (u on the
    padding indices 10..15) and n = 63"""
    return [shuffle_item(orc, og, k, 100 + k) for k in (1, 2, 5, 42)] + [example_item(orc, og), range_item(orc, og, 10, 1), range_item(orc, og, 63, 2)]


def damaged_items(orc, og):
    s5, ex, r10, r63 = shuffle_item(orc, og, 5, 105), example_item(orc, og), range_item(orc, og, 10, 1), range_item(orc, og, 63, 2)

    def edit(it, off, data):
        b = bytearray(it.proof); b[off:off + len(data)] = data; return bytes(b)

    eb = r63.off_scalars() + 64                                          # e_blinding: flipping bit 0 keeps it canonical, every point decodes
    L0 = r10.off_scalars() + 96                                          # first L of the inner-product proof
    return [
        r63.replace("flipped e_blinding bit", proof=edit(r63, eb, bytes([r63.proof[eb] ^ 1]))),
        r10.replace("undecodable L", proof=edit(r10, L0, b"\xff" * 32)),
        s5.replace("zero T_1", proof=edit(s5, s5.off_T1(), bytes(32))),
        r63.replace("non-canonical t_x", proof=edit(r63, r63.off_scalars(), le(l))),
        s5.replace("truncated", proof=s5.proof[:-1]),
        ex.replace("wrong param", param=10),
        shuffle_item(orc, og, 5, 205, permutation=False, name="non-permutation"),
        r10.replace("wrong commitment", V=r63.V),
    ]


def check_batch(bp, gpu_ctx, gens, orc, og, items, seed=bytes(32)):
    got = bp.r1cs_verify_batch(gpu_ctx, gens, [it.batch_item(bp) for it in items], ext_seed=seed)
    want = [it.expected(orc, og) for it in items]
    assert got == want, [(it.name, g, w) for it, g, w in zip(items, got, want) if g != w]
    return got


@pytest.mark.gpu
def test_mixed_batch_all_valid_then_each_damage(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 128, 1); og = orc.gens(128, 1)
    valid, damaged = valid_items(orc, og), damaged_items(orc, og)
    assert check_batch(bp, gpu_ctx, gens, orc, og, valid) == [OK] * len(valid)
    want_codes = {"truncated": FORMAT_ERROR, "non-canonical t_x": FORMAT_ERROR}
    for d in damaged:                                                   # one damaged copy at a time, in the middle of the valid proofs
        items = valid[:3] + [d] + valid[3:]
        got = check_batch(bp, gpu_ctx, gens, orc, og, items)
        assert got[3] == want_codes.get(d.name, VERIFICATION_ERROR) and got[:3] + got[4:] == [OK] * len(valid), d.name
    got = check_batch(bp, gpu_ctx, gens, orc, og, damaged + valid + damaged)     # every damage at once, twice
    assert got[len(damaged):len(damaged) + len(valid)] == [OK] * len(valid)
    gens.close()


@pytest.mark.gpu
def test_batch_of_one_equals_verify(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 128, 1); og = orc.gens(128, 1)
    for i, it in enumerate(valid_items(orc, og) + damaged_items(orc, og)):
        seed = bytes([i]) * 32
        one = bp.r1cs_verify_batch(gpu_ctx, gens, [it.batch_item(bp)], ext_seed=seed)
        assert one == [bp.r1cs_verify(gpu_ctx, gens, it.bp_transcript(bp), it.gadget, it.V, it.proof, param=it.param, ext_seed=seed)] == [it.expected(orc, og)], it.name
    gens.close()


@pytest.mark.gpu
def test_permuting_the_batch_permutes_the_verdicts(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 128, 1); og = orc.gens(128, 1)
    items = valid_items(orc, og) + damaged_items(orc, og)
    base = check_batch(bp, gpu_ctx, gens, orc, og, items)
    rnd = random.Random(3)
    for _ in range(3):
        perm = list(range(len(items))); rnd.shuffle(perm)
        got = bp.r1cs_verify_batch(gpu_ctx, gens, [items[p].batch_item(bp) for p in perm], ext_seed=bytes([7]) * 32)
        assert got == [base[p] for p in perm]
    gens.close()


@pytest.mark.gpu
def test_gens_too_small_for_one_proof(gpu_ctx, orc):
    """capacity 64: the 42-shuffle (82 multipliers, padded_n = 128) gets InvalidGeneratorsLength, every other proof is still decided"""
    import bulletproofs_b200 as bp
    og128 = orc.gens(128, 1)
    items = valid_items(orc, og128) + [damaged_items(orc, og128)[-1]]
    gens = bp.Gens(gpu_ctx, 64, 1); og = orc.gens(64, 1)
    got = check_batch(bp, gpu_ctx, gens, orc, og, items)
    assert [g for it, g in zip(items, got) if it.name == "shuffle42"] == [INVALID_GENERATORS_LENGTH]
    assert [g for it, g in zip(items, got) if it.name not in ("shuffle42", "wrong commitment")] == [OK] * (len(items) - 2) and got[-1] == VERIFICATION_ERROR
    gens.close()


@pytest.mark.gpu
def test_undecodable_point_does_not_force_the_reject_path(gpu_ctx, orc):
    """a proof with an undecodable point is left out of the combination: the batch costs the launches of an all-valid batch, where
    a proof that is merely wrong costs the per-proof re-check"""
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 128, 1); og = orc.gens(128, 1)
    valid = valid_items(orc, og); d = {it.name: it for it in damaged_items(orc, og)}

    def launches(items):
        n0 = gpu_ctx.launches
        check_batch(bp, gpu_ctx, gens, orc, og, items)
        return gpu_ctx.launches - n0

    ok = launches(valid + [valid[-1]])
    assert launches(valid + [d["undecodable L"]]) == ok
    wrong = launches(valid + [d["non-permutation"]])
    assert ok == wrong == 0 or wrong > ok                               # the mock engine counts no launches
    gens.close()


def _many(orc, og, k, count, bad_at, n_valid=4):
    valid = [shuffle_item(orc, og, k, 300 + s) for s in range(n_valid)]
    bad = [shuffle_item(orc, og, k, 400, permutation=False, name="non-permutation"),
           shuffle_item(orc, og, k, 301).replace("flipped bit", proof=bytes(b ^ (1 if i == 1 + 32 * 11 + 3 else 0) for i, b in enumerate(shuffle_item(orc, og, k, 301).proof)))]
    items = [valid[i % n_valid] for i in range(count)]
    for j, i in enumerate(bad_at):
        items[i] = bad[j % 2]
    return items


@pytest.mark.gpu
@pytest.mark.parametrize("bad_at", [(), (737,), (3, 100, 333, 334, 500, 640, 777, 901, 1023)], ids=["all-valid", "one-bad", "bad-in-many-chunks"])
def test_1024_shuffles(gpu_ctx, orc, bad_at):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 16, 1); og = orc.gens(16, 1)                  # 8-shuffle: 14 multipliers, padded_n = 16
    items = _many(orc, og, 8, 1024, bad_at)
    got = check_batch(bp, gpu_ctx, gens, orc, og, items, seed=bytes(range(32)))
    assert [i for i, g in enumerate(got) if g != OK] == list(bad_at)
    gens.close()


@pytest.mark.gpu
def test_four_shuffles_of_2049_inputs_one_bad(gpu_ctx, orc):
    """4096 multipliers per proof: the G/H sum runs over 32 index tiles of one chunk"""
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 4096, 1); og = orc.gens(4096, 1)
    items = _many(orc, og, 2049, 4, (2,), n_valid=1)
    assert check_batch(bp, gpu_ctx, gens, orc, og, items) == [OK, OK, VERIFICATION_ERROR, OK]
    gens.close()


@pytest.mark.gpu
@pytest.mark.parametrize("big_valid", [True, False], ids=["big-valid", "big-damaged"])
def test_reject_path_in_slices_with_a_2049_input_shuffle(gpu_ctx, orc, E, big_valid):
    """600 proofs whose largest has padded_n = 4096: the reject path re-checks them in two slices, [0, 512) and [512, 600), so the
    second slice's rows, G/H sums and verdicts start at proof 512.  Bad proofs on both sides of the slice boundary and last; the
    2049-input shuffle (4096 multipliers) sits in the second slice among 8-input shuffles (padded_n = 16)."""
    import bulletproofs_b200 as bp
    count, big_at, bad_at = 600, 550, (3, 511, 512, 599)
    per = r1cs_slice(E, count, 4096)
    assert per == 512 and (count + per - 1) // per == 2 and big_at // per == 1, "the slice rule moved: update the layout of this test"
    gens = bp.Gens(gpu_ctx, 4096, 1); og = orc.gens(4096, 1)
    items = _many(orc, og, 8, count, bad_at)
    big = shuffle_item(orc, og, 2049, 300)
    if not big_valid:
        flip = big.off_scalars() + 3                                       # t_x, still canonical: only the mega-check can reject it
        big = big.replace("flipped t_x bit", proof=bytes(b ^ (1 if i == flip else 0) for i, b in enumerate(big.proof)))
    items[big_at] = big
    want_of = {}
    for it in items:                                                     # the oracle's verdict of each distinct proof
        if id(it) not in want_of:
            want_of[id(it)] = it.expected(orc, og)
    want = [want_of[id(it)] for it in items]
    assert [i for i, w in enumerate(want) if w != OK] == sorted(bad_at + (() if big_valid else (big_at,)))
    got = bp.r1cs_verify_batch(gpu_ctx, gens, [it.batch_item(bp) for it in items], ext_seed=bytes(range(32)))
    assert got == want, [(i, it.name, g, w) for i, (it, g, w) in enumerate(zip(items, got, want)) if g != w]
    gens.close()


# ---------------------------------------------------------------------------------------------------------------------- CPU tier
@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_recheck_slice.argtypes = [ctypes.c_uint32] * 3; E.emul_recheck_slice.restype = ctypes.c_uint32
    return E


def r1cs_slice(E, np_, Nmax):
    """proofs per slice of the R1CS reject path: the shared slice rule with 2 * Nmax G/H entries per proof and a budget of 2^22"""
    return E.emul_recheck_slice(np_, 2 * Nmax, 1 << 22)


def _gh_reference(proofs, weighted, chunk, Nmax):
    """sum over each chunk's proofs of W g_i and W h_i (verifier.rs:409-442), W = rho u1 or u1, with Python integers"""
    rows = []
    for c0 in range(0, len(proofs), chunk):
        G, H = [0] * Nmax, [0] * Nmax
        for (N, n1, n, ch, wL, wR, wO) in proofs[c0:c0 + chunk]:
            x, yinv, u, a, b, rho, s0 = ch[:7]; usq = ch[7:]; k = N.bit_length() - 1
            s = []
            for i in range(N):
                v = s0
                for bit in range(k):
                    if i >> bit & 1:
                        v = v * usq[k - 1 - bit] % l
                s.append(v)
            for i in range(N):
                W = (rho if weighted else 1) * (1 if i < n1 else u)
                yi = pow(yinv, i, l)
                wl, wr, wo = (wL[i], wR[i], wO[i]) if i < n else (0, 0, 0)
                G[i] += W * (x * yi * wr - a * s[i])
                H[i] += W * (yi * (x * wl + wo - b * s[N - 1 - i]) - 1)
        rows.append([g % l for g in G] + [h % l for h in H])
    return rows


def test_weighted_gh_sums_against_python_integers(E):
    rnd = random.Random(11)
    # (padded_n, n1, n): k = 0 (padded_n = 1, with and without a multiplier), padding indices with u (n1 <= n < padded_n), two-phase
    # circuits, and sizes whose k splits unevenly between the low and high index tables
    shapes = [(1, 0, 0), (1, 1, 1), (2, 1, 2), (16, 5, 10), (16, 16, 16), (64, 10, 63), (8, 0, 8), (4, 2, 3), (1, 0, 1), (32, 20, 20), (128, 40, 82)]
    proofs = []
    for j in range(37):                                                   # ragged last chunk for every chunk size below
        N, n1, n = shapes[j % len(shapes)] if j < 30 else shapes[rnd.randrange(len(shapes))]
        ch = [rnd.randrange(l) for _ in range(7 + N.bit_length() - 1)]
        proofs.append((N, n1, n, ch, [rnd.randrange(l) for _ in range(n)], [rnd.randrange(l) for _ in range(n)], [rnd.randrange(l) for _ in range(n)]))
    for sub in (proofs[:1], proofs[:3], proofs):
        Nmax = max(p[0] for p in sub)
        dims = (ctypes.c_uint32 * (4 * len(sub)))(*[v for p in sub for v in (p[0], p[1], p[2], 0)])
        chal = b"".join(le(v) for p in sub for v in p[3])
        wL, wR, wO = (b"".join(le(v) for p in sub for v in p[idx]) for idx in (4, 5, 6))
        for chunk in (1, 5, 32):
            for weighted in (1, 0):
                nch = (len(sub) + chunk - 1) // chunk
                out = ctypes.create_string_buffer(32 * nch * 2 * Nmax)
                E.emul_r1cs_gh_sums(len(sub), dims, chal, wL or None, wR or None, wO or None, weighted, chunk, out)
                got = [[int.from_bytes(out.raw[32 * (r * 2 * Nmax + e):32 * (r * 2 * Nmax + e + 1)], "little") for e in range(2 * Nmax)] for r in range(nch)]
                assert got == _gh_reference(sub, weighted, chunk, Nmax), (len(sub), chunk, weighted)


def test_r1cs_tables_split_every_k(E):
    """the low/high index tables have 3 * 2^kl + 6 * 2^kh entries, kl = ceil(k/2) (the range-proof head's split)"""
    for k in range(0, 21):
        kl = (k + 1) // 2
        assert E.emul_r1cs_tab_size(k) == 3 * (1 << kl) + 6 * (1 << (k - kl))


def test_reject_path_slice_rule(E):
    """r1cs_recheck re-checks as many proofs at a time as 2^22 generator-index sums hold (2 * Nmax per proof), at least one proof
    and at most 65535 (the slice is a grid's y extent)"""
    f = lambda np_, Nmax: r1cs_slice(E, np_, Nmax)
    assert (f(600, 4096), f(70000, 1), f(10, 1 << 21)) == (512, 65535, 1)
    assert (f(3, 16), f(512, 4096), f(513, 4096), f(1 << 20, 16), f(1, 1 << 22)) == (3, 512, 512, 65535, 1)
    for np_ in (1, 2, 511, 512, 513, 600, 65535, 65536, 70000, 1 << 20):
        for lg in range(0, 23):
            assert f(np_, 1 << lg) == min(np_, 65535, max(1, (1 << 22) // (2 << lg))), (np_, lg)


def test_batch_tests_through_the_mock_engine(built):
    """this file's GPU tests against the mock engine, minus the 4096-multiplier one (the mock's MSMs are single-threaded CPU code)"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_engine"))
    import build_mock_r1cs
    build_mock_r1cs.build()
    env = dict(os.environ, BP_TEST_R1CS_MOCK="1")
    env.pop("BP_TEST_MOCK_ENGINE", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_r1cs_batch.py", "-m", "gpu", "-x", "-q", "-k", "not 2049", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    tail = "\n".join(r.stdout.splitlines()[-15:])
    assert r.returncode == 0, tail + r.stderr[-2000:]
    n_passed = int(tail.split(" passed")[0].split()[-1])
    assert n_passed >= 7, tail
