"""GPU tier (-m gpu): bp.MixedVerifier.run_device / run_device_each, mixed-geometry verification whose inputs are device buffers (torch CUDA
tensors of bp.pack_mixed's arrays), placed in the reserved mix on the device.  Verdicts are compared with the oracle's verdict of each
proof alone and with bp.verify_mixed(_each) on the same items on a context without a reserved mix.  The mix is a block of confidential
transactions, (64, m) for m in 1, 2, 4, 8."""
import random

import pytest

from test_gpu_geometry import LABEL, _cell
from test_gpu_mixed_service import FULL, MIX, _damaged, oracle, tx
from test_gpu_per_proof_transcripts import _contexts, _prove, malformed_record

pytestmark = pytest.mark.gpu

KEYS = list(MIX)


@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


@pytest.fixture(scope="module")
def gens(gpu_ctx):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 32)
    yield g
    g.close()


def _dev(data, shift):
    """bytes as a CUDA tensor whose content starts `shift` bytes into it: (tensor, address of the content)"""
    import torch
    t = torch.zeros(len(data) + shift + 8, dtype=torch.uint8)
    if data:
        t[shift:shift + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8)
    t = t.cuda()
    return t, t.data_ptr() + shift


class Call:
    """one call's inputs uploaded once (pack_mixed, every array `shift` bytes into its tensor, the proofs `base` bytes into theirs with the
    offsets moved by as much), its verdict tensor and pinned class flags"""

    def __init__(self, items, records=None, shift=0, base=0):
        import torch
        import bulletproofs_b200 as bp
        proofs, poff, ns, commitments, coff = bp.pack_mixed(items)
        poff = type(poff)("Q", [o + base for o in poff])
        self.count, self.proof_bytes, self.n_commitments = len(items), len(proofs) + base, len(commitments) // 32
        self.keep = []
        def up(b):
            t, a = _dev(b, shift)
            self.keep.append(t)
            return a
        self.proofs, self.poff, self.n = up(bytes(base) + proofs), up(poff.tobytes()), up(ns.tobytes())
        self.commitments, self.coff = up(commitments), up(coff.tobytes())
        self.records = up(b"".join(records)) if records else None
        self.verdicts = torch.zeros(len(items), dtype=torch.int32, device="cuda")
        self.flags = torch.full((len(MIX),), 7, dtype=torch.int32).pin_memory()
        torch.cuda.synchronize()

    def queue(self, v, seed):
        import bulletproofs_b200 as bp
        args = (self.proofs, self.proof_bytes, self.poff, self.n, self.commitments, self.n_commitments, self.coff, self.count, self.verdicts.data_ptr(),
                self.flags.data_ptr())
        if self.records is not None:
            v.run_device_each(self.records, *args, seed=seed)
        else:
            v.run_device(bp.Transcript(LABEL), *args, seed=seed)

    def result(self):
        """(verdicts as u32, class flags), after the context's stream has run the call"""
        return [x & 0xFFFFFFFF for x in self.verdicts.cpu().tolist()], self.flags.tolist()


class Dev:
    """a context of its own with the mix reserved"""

    def __init__(self):
        import bulletproofs_b200 as bp
        self.ctx = bp.Context(0)
        self.gens = bp.Gens(self.ctx, 64, 32)
        self.v = bp.MixedVerifier(self.ctx, self.gens, MIX)

    def run(self, items, seed, records=None, shift=0, base=0):
        """(verdicts, flags, launch delta) of one synchronised device call"""
        call = Call(items, records, shift, base)
        l0 = self.ctx.launches
        call.queue(self.v, seed)
        dl = self.ctx.launches - l0
        self.ctx.synchronize()
        return (*call.result(), dl)

    def close(self):
        self.gens.close()
        self.ctx.close()


@pytest.fixture(scope="module")
def dev():
    d = Dev()
    yield d
    d.close()


def expect(bp, orc, og, ref_ctx, ref_gens, items, seed, records=None):
    """the oracle's verdicts, checked equal to verify_mixed(_each)'s on a context without a reserved mix"""
    if records:
        direct = bp.verify_mixed_each(ref_ctx, ref_gens, [(bp.Transcript(state=t), p, V, n) for t, (p, V, n) in zip(records, items)], seed=seed)
    else:
        direct = bp.verify_mixed(ref_ctx, ref_gens, bp.Transcript(LABEL), items, seed=seed)
    want = oracle(orc, og, items, records)
    assert direct == want
    return want


def class_of(item):
    p, V, n = item
    return KEYS.index((n, len(V) // 32)) if (n, len(V) // 32) in KEYS else None


def test_full_and_partial_fill(gpu_ctx, orc, og, gens, dev):
    import bulletproofs_b200 as bp
    rnd = random.Random(1)
    for counts in (FULL, {1: 40, 2: 7, 4: 33, 8: 1}, {1: 1}):
        items = tx(orc, og, counts, rnd)
        got, flags, _ = dev.run(items, bytes([1]) * 32)
        assert got == expect(bp, orc, og, gpu_ctx, gens, items, bytes([1]) * 32) == [0] * len(items)
        assert flags == [1, 1, 1, 1]


def test_per_proof_records(gpu_ctx, orc, og, gens, dev):
    """distinct valid records per proof, and malformed ones (pos >= 166, pos_begin > pos), which give FormatError"""
    import bulletproofs_b200 as bp
    rnd = random.Random(2)
    ctxs = _contexts(orc)
    records, items = [], []
    for c, m in enumerate((1, 1, 2, 4, 8, 1, 2)):
        t = ctxs[c % len(ctxs)]
        proofs, Vs = _prove(orc, og, t, 64, m, 3, 900 + c)
        plen = len(proofs) // 3
        for i in range(3):
            records.append(t)
            items.append((proofs[i * plen:(i + 1) * plen], Vs[32 * m * i:32 * m * (i + 1)], 64))
    records[3], records[8], records[14] = malformed_record(rnd, 0), malformed_record(rnd, 1), malformed_record(rnd, 0)
    perm = list(range(len(items)))
    rnd.shuffle(perm)
    items, records = [items[i] for i in perm], [records[i] for i in perm]
    got, flags, _ = dev.run(items, bytes([2]) * 32, records=records)
    assert got == expect(bp, orc, og, gpu_ctx, gens, items, bytes([2]) * 32, records)
    assert sorted(v for v in got if v) == [2, 2, 2] and flags == [1, 1, 1, 1]


def test_per_proof_parameter_codes(gpu_ctx, orc, og, gens, dev):
    """wrong length, n outside {8, 16, 32, 64}, m = 0, n m != 2^k, more parties than the table, a rejected proof with a non-canonical
    scalar: each proof keeps verify_mixed's code among valid proofs of the mix"""
    import bulletproofs_b200 as bp
    rnd = random.Random(3)
    valid = tx(orc, og, {1: 4, 2: 3, 4: 2})
    p, V, _ = valid[0]
    p4, V4, _ = valid[-1]
    nc = bytearray(p4[:-64])                                       # length of n m = 2, with a non-canonical t_x
    nc[128:160] = b"\xff" * 32
    odd = [(p[:-1], V, 64), (p, V, 12), (p, b"", 64), (p4, V4[:96], 64), (p + bytes(64 * 6), V * 64, 64), (bytes(nc), V4, 64), (p, V * 2, 64)]
    items = valid + odd
    rnd.shuffle(items)
    got, flags, _ = dev.run(items, bytes([3]) * 32)
    want = expect(bp, orc, og, gpu_ctx, gens, items, bytes([3]) * 32)
    assert got == want and flags == [1, 1, 1, 1]
    assert sorted(set(want)) == [0, 1, 2, 3, 4]


def test_unplaced_proofs(gpu_ctx, orc, og, gens, dev):
    """a class outside the mix and a class over capacity: BP_VERDICT_UNPLACED on exactly those proofs (every one of the unreserved class,
    the later ones in input order of the over-full class), the verify_mixed verdict everywhere else"""
    import bulletproofs_b200 as bp
    rnd = random.Random(4)
    proofs, Vs, plen = _cell(orc, og, 32, 2)
    other = [(proofs[i * plen:(i + 1) * plen], Vs[64 * i:64 * (i + 1)], 32) for i in range(5)]
    items = tx(orc, og, {1: 10, 2: 40, 8: 3}) + other
    rnd.shuffle(items)
    got, flags, _ = dev.run(items, bytes([4]) * 32)
    seen, unplaced = {}, []
    for i, it in enumerate(items):
        c = class_of(it)
        seen[c] = seen.get(c, 0) + 1
        if c is None or seen[c] > MIX[KEYS[c]]:
            unplaced.append(i)
    assert len(unplaced) == 5 + 7
    assert [i for i, v in enumerate(got) if v == bp.VERDICT_UNPLACED] == unplaced
    want = expect(bp, orc, og, gpu_ctx, gens, items, bytes([4]) * 32)
    assert [g for i, g in enumerate(got) if i not in unplaced] == [w for i, w in enumerate(want) if i not in unplaced]
    assert flags == [1, 1, 1, 1]


def test_damaged_classes_are_flagged(gpu_ctx, orc, og, gens, dev):
    """damage in one class, then in three: only those classes' flags are 0, their well-formed proofs are VerificationError, the other
    classes are exact, and verify_mixed on the flagged classes' proofs gives the oracle's verdicts"""
    import bulletproofs_b200 as bp
    rnd = random.Random(5)
    for ms in ((4,), (1, 2, 8)):
        items, _ = _damaged(orc, og, ms, rnd)
        got, flags, _ = dev.run(items, bytes([5]) * 32)
        want = oracle(orc, og, items)
        assert flags == [0 if m in ms else 1 for _, m in KEYS]
        for i, it in enumerate(items):
            flagged = not flags[class_of(it)]
            assert got[i] == ((1 if want[i] == 0 else want[i]) if flagged else want[i]), (i, got[i], want[i])
        redo = [i for i, it in enumerate(items) if not flags[class_of(it)]]
        again = bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), [items[i] for i in redo], seed=bytes([5]) * 32)
        assert again == [want[i] for i in redo]


def test_calls_queued_back_to_back(gpu_ctx, orc, og, gens, dev):
    """four calls at different fills, one with damage and one with records, queued on one context before one synchronise: each gets its
    own verdicts and flags"""
    import bulletproofs_b200 as bp
    rnd = random.Random(6)
    damaged, _ = _damaged(orc, og, (2,), rnd)
    ctxs = _contexts(orc)
    proofs, Vs = _prove(orc, og, ctxs[1], 64, 4, 5, 950)
    plen = len(proofs) // 5
    rec_items = [(proofs[i * plen:(i + 1) * plen], Vs[128 * i:128 * (i + 1)], 64) for i in range(5)]
    specs = [(tx(orc, og, FULL, rnd), None), (damaged, None), (tx(orc, og, {1: 3, 8: 2}, rnd), None), (rec_items, [ctxs[1]] * 5)]
    calls = [Call(items, records) for items, records in specs]
    for k, c in enumerate(calls):
        c.queue(dev.v, bytes([6 + k]) * 32)
    dev.ctx.synchronize()
    for k, ((items, records), c) in enumerate(zip(specs, calls)):
        got, flags = c.result()
        want = oracle(orc, og, items, records)
        if k == 1:
            assert flags == [1, 0, 1, 1]
            assert all(g == (w if w > 1 else (1 if class_of(it) == 1 else w)) for g, w, it in zip(got, want, items))
        else:
            assert got == want == [0] * len(items) and flags == [1, 1, 1, 1]


def test_stale_slots_have_no_effect(gpu_ctx, orc, og, gens, dev):
    """a full call with an invalid proof in the last (64, 2) slot (its class is flagged, every proof of it VerificationError), then a call
    with fewer (64, 2) proofs, all valid: every one accepted"""
    import bulletproofs_b200 as bp
    items = tx(orc, og, FULL)
    i = FULL[1] + FULL[2] - 1
    p, V, n = items[i]
    pb = bytearray(p)
    pb[128] ^= 1
    items[i] = (bytes(pb), V, n)
    got, flags, _ = dev.run(items, bytes([7]) * 32)
    assert got == [1 if FULL[1] <= j <= i else 0 for j in range(len(items))] and flags == [1, 0, 1, 1]
    got, flags, _ = dev.run(tx(orc, og, {1: 10, 2: 20, 4: 2}), bytes([7]) * 32)
    assert got == [0] * 32 and flags == [1, 1, 1, 1]


def test_inputs_at_odd_byte_offsets(gpu_ctx, orc, og, gens, dev):
    """every input array at an odd address, and proof offsets that do not start at 0"""
    import bulletproofs_b200 as bp
    items = tx(orc, og, {1: 20, 2: 9, 4: 5, 8: 2}, random.Random(8))
    items[4] = (items[4][0][:-32], items[4][1], 64)
    ctxs = _contexts(orc)
    for shift, base in ((1, 0), (3, 77)):
        got, flags, _ = dev.run(items, bytes([8]) * 32, shift=shift, base=base)
        assert got == expect(bp, orc, og, gpu_ctx, gens, items, bytes([8]) * 32) and flags == [1, 1, 1, 1]
    proofs, Vs = _prove(orc, og, ctxs[2], 64, 2, 4, 960)
    plen = len(proofs) // 4
    rec_items = [(proofs[i * plen:(i + 1) * plen], Vs[64 * i:64 * (i + 1)], 64) for i in range(4)]
    got, _, _ = dev.run(rec_items, bytes([8]) * 32, records=[ctxs[2]] * 4, shift=5, base=3)
    assert got == [0] * 4


def test_argument_errors_queue_nothing(gpu_ctx, orc, og, gens, dev):
    """no mix, another table, a NULL pointer, count 0, count >= 2^24, misaligned verdicts and a pending begin are refused without a launch;
    after finish the device call works, and so does a reserved BatchVerifier on the same context"""
    import bulletproofs_b200 as bp
    items = tx(orc, og, {1: 3, 2: 1})
    call = Call(items)
    L = bp.lib()
    def raw(ctx, g, count=call.count, proofs=call.proofs, verdicts=call.verdicts.data_ptr()):
        return L.bp_rangeproof_verify_mixed_device(ctx._h, g._h, bp.Transcript(LABEL).to_bytes(), count, proofs, call.proof_bytes, call.poff, call.n,
                                                   call.commitments, call.n_commitments, call.coff, None, verdicts, None)
    plain = bp.Context(0)
    plain_gens = bp.Gens(plain, 64, 32)
    other = bp.Gens(dev.ctx, 64, 32)
    try:
        cases = [(plain, plain_gens, {}), (dev.ctx, other, {}), (dev.ctx, dev.gens, {"proofs": None}), (dev.ctx, dev.gens, {"count": 0}),
                 (dev.ctx, dev.gens, {"count": 1 << 24}), (dev.ctx, dev.gens, {"verdicts": call.verdicts.data_ptr() + 2})]
        for ctx, g, kw in cases:
            l0 = ctx.launches
            assert raw(ctx, g, **kw) == bp.ERR_INVALID_ARGUMENT
            assert ctx.launches == l0
        dev.v.begin(bp.Transcript(LABEL), items, seed=bytes([9]) * 32)
        l0 = dev.ctx.launches
        assert raw(dev.ctx, dev.gens) == bp.ERR_INVALID_ARGUMENT and dev.ctx.launches == l0
        assert dev.v.finish() == [0] * 4
        call.queue(dev.v, bytes([9]) * 32)
        dev.ctx.synchronize()
        assert call.result() == ([0] * 4, [1, 1, 1, 1])
        proofs, Vs, plen = _cell(orc, og, 64, 1)
        bv = bp.BatchVerifier(dev.ctx, dev.gens, bp.Transcript(LABEL), 64, 1, 8)
        import ctypes
        pb, vb = ctypes.create_string_buffer(proofs[:8 * plen]), ctypes.create_string_buffer(Vs[:8 * 32])
        bv.begin(ctypes.addressof(pb), ctypes.addressof(vb), seed=bytes([9]) * 32)
        assert list(bv.finish()) == [0] * 8
        got, _, _ = dev.run(items, bytes([9]) * 32)
        assert got == [0] * 4
    finally:
        other.close()
        plain_gens.close()
        plain.close()


def test_launches_do_not_depend_on_count(gpu_ctx, orc, og, gens, dev):
    """1, 1000 and 8192 proofs (the last two mostly unplaced) cost the same launches, the planner kernels, one gather, the graph and one
    verdict kernel"""
    import bulletproofs_b200 as bp
    rnd = random.Random(10)
    deltas = []
    for count in (1, 1000, 8192):
        items = tx(orc, og, {1: count}, rnd) if count == 1 else tx(orc, og, {m: count // 4 for m in (1, 2, 4, 8)}, rnd)
        got, flags, dl = dev.run(items, bytes([10]) * 32)
        deltas.append(dl)
        placed = [v for v in got if v != bp.VERDICT_UNPLACED]
        assert placed == [0] * min(len(items), sum(MIX.values())) and flags == [1, 1, 1, 1]
    assert deltas[0] == deltas[1] == deltas[2] > 0
