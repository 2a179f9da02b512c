"""CPU tier: the per-proof caller state of the range-proof transcript replay (rp_transcript_proof, what k_rp_transcript runs for proof p),
compiled for the host by tests/host_emul.  Records packed back to back from an odd address give every proof the raw challenge rows of
the scheduled replay from an aligned copy of its own state (emul_rp_transcript_both, checked against the byte-wise STROBE replay by
test_transcript_sched_cpu.py), and a record no Merlin transcript can hold between operations (pos at or beyond the 166-byte rate, or
pos_begin above pos) gives FormatError before the replay writes a row."""
import ctypes
import os
import random

import pytest

from test_transcript_sched_cpu import caller_states, random_proof, replay

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REC = 203
FORMAT_ERROR = 2


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    e.emul_rp_transcript_both.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32,
                                          ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    e.emul_rp_transcript_proof.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p,
                                           ctypes.c_uint64, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_char_p]
    return e


def packed(records, front):
    """the records back to back from byte `front` of a buffer that ends with the last record; (buffer, address of record 0)"""
    buf = ctypes.create_string_buffer(front + REC * len(records))
    ctypes.memmove(ctypes.addressof(buf) + front, b"".join(records), REC * len(records))
    return buf, ctypes.addressof(buf) + front


def run(E, proof, k, V, n, m, base, stride, p, seed):
    raw = ctypes.create_string_buffer(b"\xa5" * 64 * (6 + k), 64 * (6 + k))
    st = E.emul_rp_transcript_proof(bytes(proof), k, V, n, m, base, stride, p, seed, raw)
    return st, raw.raw


@pytest.mark.parametrize("n,m,front", [(64, 1, 1), (8, 4, 3), (32, 2, 8), (16, 8, 5)])
def test_records_at_any_address_replay_their_own_state(E, n, m, front):
    rnd = random.Random(100 * n + m + front)
    k = (n * m).bit_length() - 1
    states = caller_states(E, rnd)
    rnd.shuffle(states)
    buf, base = packed(states, front)
    seed = rnd.randbytes(32)
    for p, tstate in enumerate(states):
        proof, V = random_proof(rnd, k), rnd.randbytes(32 * m)
        _, ss, _, want = replay(E, proof, k, V, n, m, tstate, seed)
        st, got = run(E, proof, k, V, n, m, base, REC, p, seed)
        assert st == ss == 0 and got == want, (p, tstate[200], tstate[201])
        single, addr = packed([tstate], 0)              # stride 0: every proof from the one state
        assert run(E, proof, k, V, n, m, addr, 0, 7, seed) == (0, want)


def malformed_records(rnd):
    out = [rnd.randbytes(200) + bytes([pos, rnd.randrange(0, 256), rnd.randrange(256)]) for pos in range(166, 256)]
    out += [rnd.randbytes(200) + bytes([pos, rnd.randrange(pos + 1, 256), rnd.randrange(256)]) for pos in range(0, 166, 5)]
    return out


def test_malformed_records_are_format_errors(E):
    """each malformed record as the last one of an exactly sized buffer at an odd address, between well-formed records: FormatError and
    no row written for it, the rows of its neighbours unchanged"""
    rnd = random.Random(5)
    n, m, k = 64, 2, 7
    good = caller_states(E, rnd)[:3]
    seed, V = rnd.randbytes(32), rnd.randbytes(64)
    proof = random_proof(rnd, k)
    want = [replay(E, proof, k, V, n, m, t, seed)[3] for t in good]
    untouched = b"\xa5" * 64 * (6 + k)
    for bad in malformed_records(rnd):
        recs = [good[0], good[1], bad, good[2], bad]
        buf, base = packed(recs, 1)
        got = [run(E, proof, k, V, n, m, base, REC, p, seed) for p in range(len(recs))]
        assert got[2] == got[4] == (FORMAT_ERROR, untouched), (bad[200], bad[201])
        assert [got[0], got[1], got[3]] == [(0, w) for w in want]


def test_proof_verdicts_beside_records(E):
    """a non-canonical scalar gives FormatError under a well-formed record as under a malformed one; a well-formed record leaves the
    proof's own VerificationError and its rows as they are"""
    rnd = random.Random(6)
    n, m, k = 16, 1, 4
    good, bad = caller_states(E, rnd)[2], malformed_records(rnd)[0]
    buf, base = packed([good, bad], 7)
    V, seed = rnd.randbytes(32), rnd.randbytes(32)
    proof = random_proof(rnd, k); proof[160 + 31] = 0xFF
    assert run(E, proof, k, V, n, m, base, REC, 0, seed)[0] == FORMAT_ERROR
    assert run(E, proof, k, V, n, m, base, REC, 1, seed)[0] == FORMAT_ERROR
    proof = random_proof(rnd, k); proof[0:32] = bytes(32)             # identity A: VerificationError, rows still written
    st, raw = run(E, proof, k, V, n, m, base, REC, 0, seed)
    assert st == 1 and raw == replay(E, proof, k, V, n, m, good, seed)[3]
