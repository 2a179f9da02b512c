"""CPU tier: the C-ABI library loads and exports every symbol include/bpmsm.h declares; the host-only
helpers (Merlin transcript) behave like the oracle's; a compute call without a GPU fails loudly."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "bpmsm.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bp_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound(built):
    import bulletproofs_b200 as bp
    L = bp.lib()
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(L, name), f"{name} declared in bpmsm.h but not exported by libbpmsm.so"
        assert name in bp.SYMBOLS, f"{name} has no ctypes signature in bulletproofs_b200.SYMBOLS"
    assert set(bp.SYMBOLS) <= set(declared)
    assert set(bp.TEST_HOOKS) <= set(declared)
    for name in bp.TEST_HOOKS:                  # bound with their signatures, like every product symbol
        assert list(getattr(L, name).argtypes) == list(bp.SYMBOLS[name][1]), name


def test_transcript_helpers_match_oracle(built, orc):
    import bulletproofs_b200 as bp
    t = bp.Transcript(b"test protocol")
    t.append_message(b"some label", b"some data")
    assert t.challenge_bytes(b"challenge", 32).hex() == "d5a21972d0d5fe320c0d263fac7fffb8145aa640af6e9bca177c03c7efcf0615"
    for label in (b"", b"x", b"Deserialize-And-Verify Test", bytes(range(200))):
        assert bp.Transcript(label).to_bytes() == orc.transcript(label)[:bp.TRANSCRIPT_BYTES]
    t = bp.Transcript(b"abc"); st = orc.transcript(b"abc")
    for i in range(12):                      # cross the 166-byte rate several times
        t.append_message(b"msg", bytes([i]) * 37); st = orc.transcript_append(st, b"msg", bytes([i]) * 37)
        t.append_u64(b"n", i * 1000003); st = orc.transcript_append(st, b"n", (i * 1000003).to_bytes(8, "little"))
        st, want = orc.transcript_challenge(st, b"c", 64)
        assert t.challenge_bytes(b"c", 64) == want
        assert t.to_bytes() == st[:bp.TRANSCRIPT_BYTES]


def test_no_cpu_fallback(built):
    """Without a usable H100 the product path must raise, never compute on the CPU."""
    import bulletproofs_b200 as bp
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        pytest.skip("GPU present: covered by the -m gpu tier")
    with pytest.raises(bp.BpError) as e:
        bp.Context(0)
    assert e.value.code == bp.ERR_CUDA
    out = ctypes.create_string_buffer(32)
    assert bp.lib().bp_msm(None, b"", b"", 0, out) == bp.ERR_INVALID_ARGUMENT
