"""CPU tier: the scheduled range-proof transcript replay (rp_tr_program + rp_transcript_sched, the form k_rp_transcript runs with
the Keccak state in registers) against the byte-wise STROBE replay (rp_transcript_raw), both compiled for the host by
tests/host_emul.  The raw challenge bytes and the verdict must be identical for every caller transcript state -- real Merlin
states, and a state at each of the 166 byte positions the caller may leave it at, so that for every geometry the positions whose
operation headers end exactly on the rate boundary are reached -- and for n*m from 8 to 2048."""
import ctypes
import os
import random

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEOMS = [(8, 1), (16, 1), (32, 1), (64, 1), (8, 2), (64, 2), (16, 8), (64, 4), (32, 16), (64, 8), (64, 16), (64, 32), (16, 128)]


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    e.emul_rp_transcript_both.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32,
                                          ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    return e


def caller_states(E, rnd):
    """Serialized caller transcripts: real Merlin states after appends of several lengths, and arbitrary states at every position
    class (pos_begin <= pos), including the positions whose next header crosses the rate boundary."""
    out = []
    for extra in (0, 1, 2, 7, 33, 100, 137):
        st = ctypes.create_string_buffer(203)
        E.emul_transcript_new(b"range proof replay", 18, st)
        if extra:
            E.emul_transcript_append(st, b"ctx", rnd.randbytes(extra), extra)
        out.append(st.raw)
    for pos in range(166):                              # every position below the rate (166)
        pb = rnd.randrange(0, pos + 1)
        out.append(rnd.randbytes(200) + bytes([pos, pb, rnd.randrange(256)]))
    return out


def random_proof(rnd, k):
    """Proof bytes with canonical scalars (top byte < 0x10) and nonzero point encodings."""
    b = bytearray(rnd.randbytes(32 * (9 + 2 * k)))
    for off in (128, 160, 192, 224 + 64 * k, 224 + 64 * k + 32):
        b[off + 31] &= 0x0F
    return b


def replay(E, proof, k, V, n, m, tstate, seed):
    rows = 6 + k
    rb, rs = ctypes.create_string_buffer(64 * rows), ctypes.create_string_buffer(64 * rows)
    st = E.emul_rp_transcript_both(bytes(proof), k, V, n, m, tstate, seed, rb, rs)
    return st & 0xFF, st >> 8, rb.raw, rs.raw


@pytest.mark.parametrize("n,m", GEOMS)
def test_sched_replay_matches_bytewise(E, n, m):
    rnd = random.Random(1000 * n + m)
    k = (n * m).bit_length() - 1
    for tstate in caller_states(E, rnd):
        proof, V, seed = random_proof(rnd, k), rnd.randbytes(32 * m), rnd.randbytes(32)
        sb, ss, rb, rs = replay(E, proof, k, V, n, m, tstate, seed)
        assert sb == ss == 0
        assert rb == rs, (n, m, tstate[200], tstate[201])


def test_sched_replay_verdicts(E):
    """A zero point encoding (VerificationError) still yields the full challenge rows; a non-canonical scalar (FormatError) stops
    both forms before any hashing."""
    rnd = random.Random(7)
    n, m, k = 64, 2, 7
    tstate = caller_states(E, rnd)[3]
    V, seed = rnd.randbytes(64), rnd.randbytes(32)
    for off in (0, 32, 64, 96, 224, 224 + 64 * 3 + 32):
        proof = random_proof(rnd, k); proof[off:off + 32] = bytes(32)
        sb, ss, rb, rs = replay(E, proof, k, V, n, m, tstate, seed)
        assert sb == ss == 1 and rb == rs, off
    proof = random_proof(rnd, k); proof[160 + 31] = 0xFF
    sb, ss, _, _ = replay(E, proof, k, V, n, m, tstate, seed)
    assert sb == ss == 2
    sb, ss, rb, rs = replay(E, random_proof(rnd, k), k, bytes(64), n, m, tstate, seed)     # identity commitments are allowed
    assert sb == ss == 0 and rb == rs
