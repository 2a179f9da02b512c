"""CPU tier of the reserved LinearProof device path (bp_linear_verify_device): the pass arithmetic of its reject loop and the record
check of the transcript replay both LinearProof forms share, compiled for the host by tests/host_emul/emul_linear_device.cpp.

- The loop runs ceil(live / P) iterations when the combined check failed and none otherwise, live clamped to the capacity, and its
  slices cover [0, live) exactly once, P = the slice rule at the capacity.
- A record no Merlin transcript can hold between operations (pos at or past the 166-byte STROBE rate, or pos_begin above pos) gives
  FormatError and writes nothing, in particular nothing past the 200-byte state; pos 165 is valid and stays inside it.
- Valid records still replay to bp.Transcript's challenges."""
import ctypes
import os

import pytest

from test_linear_verify_batch import FORMAT_ERROR, OK, _gens, _replay_python, lg, orc_proof, rng_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 512


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    for f in ("emul_lin_x_slice", "emul_lin_x_clamp", "emul_lin_x_iters", "emul_lin_x_slice_live"):
        getattr(E, f).restype = ctypes.c_uint32
    E.emul_lin_x_slice.argtypes = [ctypes.c_uint32] * 3
    E.emul_lin_x_clamp.argtypes = [ctypes.c_uint32] * 2
    E.emul_lin_x_iters.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int]
    E.emul_lin_x_slice_live.argtypes = [ctypes.c_uint32] * 3
    E.emul_lin_transcript_state.restype = ctypes.c_uint32
    E.emul_recheck_slice.argtypes = [ctypes.c_uint32] * 3; E.emul_recheck_slice.restype = ctypes.c_uint32
    return E


@pytest.mark.parametrize("n,capacity,P", [(1024, 1030, 1000), (1024, 1, 1), (1, 1 << 20, 65535), (64, 64, 64), (1 << 20, 3, 1)])
def test_slice_is_the_blocking_reject_paths_slice_at_capacity(E, n, capacity, P):
    k = lg(n)
    assert E.emul_lin_x_slice(capacity, n, k) == E.emul_recheck_slice(capacity, n + 2 + 2 + 2 * k, 1 << 20) == P


@pytest.mark.parametrize("capacity,P", [(1, 1), (32, 32), (33, 32), (1030, 1000), (1 << 20, 65535), (1 << 20, 1), (2**32 - 1, 7)])
def test_iterations_and_slices_cover_the_live_proofs_once(E, capacity, P):
    lives = {0, 1, P - 1, P, P + 1, capacity - 1, capacity, capacity + 1, 2 * capacity, 2**32 - 1} - {-1}
    for live in sorted(x for x in lives if 0 <= x < 2**32):
        c = E.emul_lin_x_clamp(live, capacity)
        assert c == min(live, capacity)
        assert E.emul_lin_x_iters(c, P, 0) == 0
        it = E.emul_lin_x_iters(c, P, 1)
        assert it == -(-c // P)
        assert it <= -(-capacity // P)
        if it > 100000:
            continue
        covered = sum(E.emul_lin_x_slice_live(i, P, c) for i in range(it))
        assert covered == c
        assert all(E.emul_lin_x_slice_live(i, P, c) == P for i in range(max(it - 1, 0)))
        assert E.emul_lin_x_slice_live(it, P, c) == 0


def _run(E, p, k, n, enc, record, seed):
    raw = ctypes.create_string_buffer(b"\x5a" * 64 * (k + 2), 64 * (k + 2))
    state = ctypes.create_string_buffer(b"\xc3" * (200 + GUARD), 200 + GUARD)
    code = E.emul_lin_transcript_state(p.proof, k, n, p.C, p.b, enc, record, seed, raw, state)
    return code, raw.raw, state.raw


@pytest.mark.parametrize("pos,pos_begin", [(166, 0), (200, 0), (255, 3), (165, 166), (40, 41), (0, 255)])
def test_malformed_records_are_format_errors_and_write_nothing(E, orc, pos, pos_begin):
    import bulletproofs_b200 as bp
    n, k = 16, 4
    G, F, B = _gens(orc, n)
    p = orc_proof(orc, G, F, B, n, 11, b"emul linear record")
    record = bp.Transcript(p.label).to_bytes()[:200] + bytes([pos, pos_begin, 0])
    code, raw, state = _run(E, p, k, n, B + F + G, record, bytes(32))
    assert code == FORMAT_ERROR
    assert raw == b"\x5a" * 64 * (k + 2) and state == b"\xc3" * (200 + GUARD)


def test_pos_at_the_last_byte_of_the_rate_stays_in_the_state(E, orc):
    """pos 165: the next absorbed byte runs the permutation, which touches st[166], st[167] and nothing past 200"""
    import bulletproofs_b200 as bp
    n, k = 16, 4
    G, F, B = _gens(orc, n)
    p = orc_proof(orc, G, F, B, n, 12, b"emul linear pos 165")
    for pos_begin in (0, 100, 165):
        record = bp.Transcript(p.label).to_bytes()[:200] + bytes([165, pos_begin, 0])
        code, raw, state = _run(E, p, k, n, B + F + G, record, bytes(32))
        assert code == OK
        assert state[200:] == b"\xc3" * GUARD


@pytest.mark.parametrize("n", [1, 2, 16, 256])
def test_valid_records_replay_to_the_python_transcript(E, orc, n):
    import bulletproofs_b200 as bp
    k = lg(n)
    G, F, B = _gens(orc, n)
    seed = bytes(range(32, 64))
    for j in range(3):
        p = orc_proof(orc, G, F, B, n, 70 + j, b"emul linear valid %d %d" % (n, j))
        code, raw, state = _run(E, p, k, n, B + F + G, bp.Transcript(p.label).to_bytes(), seed)
        assert code == OK and state[200:] == b"\xc3" * GUARD
        xs, wire = _replay_python(bp, p, n, G, F, B)
        assert [raw[64 * i:64 * i + 64] for i in range(k + 1)] == xs
        assert raw[64 * (k + 1):] == rng_bytes(wire, seed, 64, b"linear_a_r", p.proof[64 * k + 32:64 * k + 96])
