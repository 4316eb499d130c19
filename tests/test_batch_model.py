"""The whole-batch model of tests/batch_model.py against the CPU coder, and the cases the GPU batch tests
(test_batch_scale.py) use: the banks' stereo ties on the reference's own unit sizes, tiled batches through the
reference encoder and decoder, the packing-plan restatement at its two bounds and the chunk plans the host calls
reach."""
import numpy as np
import pytest

import batch_model as B
import oracle_lib as ol


@pytest.fixture(scope="module")
def O():
    return ol.best()


# ------------------------------------------------------------------------------------ banks --

def test_stereo_ties_on_the_reference_unit_sizes(O):
    """Each tie frame codes L - R to exactly its intended number of words more than R, and the reference encoder
    takes the difference only when it is strictly smaller."""
    bank = B.encode_bank(2)
    for name, (delta, sub_type) in B.TIES.items():
        f = bank.index(name)
        lft, r = bank.pcm[f, :, 0].astype(np.int32), bank.pcm[f, :, 1].astype(np.int32)
        n_r, w_r = B.unit_words(O, r)
        n_d, w_d = B.unit_words(O, lft - r)
        assert n_d - n_r == delta, name
        assert np.array_equal(w_d, w_r) == (name == "tie_same"), name
        d, words = O.encode_frames(bank.pcm[f], 2)
        assert d[1]["subframe_type"] == sub_type and d[1]["parent_channel"] == (0 if sub_type else 1), name
        one = B.tile(bank, [f])
        assert d.tobytes() == one.descs.tobytes() and np.array_equal(words, one.words), name
        rw = int(d[1]["refl_words"]) + int(d[1]["res_words"])
        assert rw == (n_d if sub_type else n_r), name


def test_banks_are_distinct_and_varied():
    for ch, lo in ((2, 90), (8, 80)):
        bank = B.encode_bank(ch)
        assert lo <= len(bank) <= 200
        flat = bank.pcm.reshape(len(bank), -1)
        assert len({row.tobytes() for row in flat}) == len(bank), ch
        # full-scale noise: the largest streams the encoder makes
        assert bank.frame_words.max() >= ch * 1000
    st = B.encode_bank(2).descs[:, 1]["subframe_type"]
    assert st.any() and not st.all()


def test_oct_bank_holds_the_golden_lossy_frames():
    """The golden frames the reference decoder does not reproduce: frame A at channel 1, frame B at channel 4,
    both from sample 1."""
    bank = B.encode_bank(8)
    rec = {(int(r["frame"]), int(r["channel"])): int(r["first_sample"]) for r in bank.records}
    assert rec[(bank.index("lossy_a"), 1)] == 1 and rec[(bank.index("lossy_b"), 4)] == 1


@pytest.mark.parametrize("ch", [2, 8])
def test_tiled_batch_is_what_the_reference_codes(O, ch):
    """About 40 frames with repeats, ties or lossy frames among them: the reference encoder on the whole batch gives
    exactly the tiled descriptors and words, and its decoder the tiled PCM and report."""
    bank = B.encode_bank(ch)
    rng = np.random.default_rng(ch)
    idx = rng.integers(0, len(bank), 40)
    special = [bank.index(n) for n in (B.TIES if ch == 2 else ("lossy_a", "lossy_b"))]
    idx[[0, 7, 8, 20, 39]] = [special[j % len(special)] for j in range(5)]
    idx[30:33] = idx[7]                                          # the same frame three times over
    want = B.tile(bank, idx, frame_base=1000)
    descs, words = O.encode_frames(want.pcm, ch)
    assert descs.tobytes() == want.descs.tobytes()
    assert np.array_equal(words, want.words) and want.used == words.size
    out = O.decode_frames(descs, words, ch)
    assert np.array_equal(out, want.decoded)
    rep = B.report_records(out, want.pcm, ch)
    rep["frame"] += 1000
    assert rep.tolist() == want.report.tolist()
    if ch == 8:
        assert want.report.size >= 5


def test_tiled_crafted_batches_are_what_the_reference_decodes(O):
    """Descriptors pointing many times at the same words of the one bank arena."""
    bank = B.decode_bank()
    assert sorted(set(bank.widths[:, 0])) == list(range(1, B.MAX_WIDTH + 1))
    idx = np.random.default_rng(3).integers(0, bank.descs.shape[0], 300)
    descs, words, pcm = bank.tile(idx)
    assert np.array_equal(O.decode_frames(descs, words, 1), pcm)
    b16 = B.frames16_bank()
    assert (b16.descs["subframe_type"] == 1).any(axis=1).sum() >= 2
    idx = np.random.default_rng(4).integers(0, b16.descs.shape[0], 7)
    descs, words, pcm = b16.tile(idx)
    assert np.array_equal(O.decode_frames(descs, words, 16), pcm)


# ----------------------------------------------------------------------------- packing plan --

def _check_bounds(counts):
    t = B.segment_templates(counts)
    n = int(sum(counts))
    assert len(t) <= B.MAX_TEMPLATES, counts
    assert B.plan_warps(t) <= B.synthesis_warps(n), counts
    placed = np.zeros(16, np.int64)                              # every subframe has exactly one place
    for rep, _, copies in t:
        placed += rep * np.array(copies)
    assert placed[1:B.MAX_WIDTH + 1].tolist() == [int(c) for c in counts]
    return len(t)


def test_template_bounds_random_and_hill_climbed():
    """Seeded random width counts, then a hill climb on the template count: never more than MAX_TEMPLATES templates
    (the shared array of k_decode_plan), never more than synthesis_warps(n) warps (the seg_index allocation)."""
    rng = np.random.default_rng(5)
    for _ in range(300):
        counts = rng.integers(0, rng.choice([3, 40, 2000, 20000]), B.MAX_WIDTH) * (rng.random(B.MAX_WIDTH) < 0.8)
        _check_bounds(counts)
    best = 0
    for _ in range(4):
        cur = rng.integers(1, 10000, B.MAX_WIDTH)
        score = _check_bounds(cur)
        for _ in range(400):
            nxt = np.maximum(cur + rng.integers(-300, 301, B.MAX_WIDTH) * (rng.random(B.MAX_WIDTH) < 0.3), 0)
            s = _check_bounds(nxt)
            if s >= score:
                cur, score = nxt, s
        best = max(best, score)
    assert best >= 20                                            # the climb gets near the bound


def test_plan_cases_reach_their_bounds():
    t = B.segment_templates(B.PLAN_26)
    assert sum(B.PLAN_26) == 93259 and len(t) == B.MAX_TEMPLATES
    assert -(-sum(B.PLAN_26) // B.SCAN_TILE) > 64 + 1           # CTAs past the plan's second 64-CTA stride
    n = sum(B.PLAN_ODD13)
    assert n % 2 == 1 and n > 65536
    assert B.plan_warps(B.segment_templates(B.PLAN_ODD13)) == B.synthesis_warps(n)
    n1 = sum(B.PLAN_WIDTH1)
    assert n1 % 32 and B.plan_warps(B.segment_templates(B.PLAN_WIDTH1)) == -(-n1 // 32)
    assert -(-B.FRAMES16 * 16 // B.SCAN_TILE) == 66
    for w in range(1, B.MAX_WIDTH + 1):
        assert all(B.width(o) == w for o in B.orders_of_width(w))


def test_device_batches_cross_the_scan_edges():
    """The one-call encode shapes: the bench's stereo batch, one past 64 scan CTAs with a partial last CTA and
    the 8-channel one; EDGE_FRAMES straddle CTA edges."""
    ctas = {(ch, n): -(-n * ch // B.SCAN_TILE) for ch, n in B.DEVICE_BATCHES}
    assert ctas == {(2, 12919): 26, (2, 33000): 65, (8, 8200): 65}
    assert 33000 * 2 % B.SCAN_TILE
    assert [2 * f for f in B.EDGE_FRAMES] == [1022, 1024, 32766, 32768]


# ------------------------------------------------------------------------------- chunk plan --

def test_chunk_plan_reaches_every_branch():
    kind = {}
    for n, forced in B.HOST_PLANS:
        start, f = B.plan_chunks(n, forced)
        assert start[0] == 0 and start[-1] == n and all(a < b for a, b in zip(start, start[1:])), (n, forced)
        assert f["chunks"] <= B.MAX_CHUNKS
        kind[(n, forced)] = f
    for n in (1, 511, 512):
        assert kind[(n, None)]["chunks"] == 1
    for n in (513, 1536):
        assert kind[(n, None)]["chunks"] > 1 and not kind[(n, None)]["taper"]
    for n in (1537, 2047):
        assert kind[(n, None)]["cut_first"] and not kind[(n, None)]["cut_last"]
    for n in (2048, 4096, 5000):
        assert kind[(n, None)]["cut_first"] and kind[(n, None)]["cut_last"]
    assert kind[(4097, None)]["chunk"] == 513
    for n, forced in ((72, 1), (500, 7)):
        assert kind[(n, forced)]["chunks"] == B.MAX_CHUNKS and not kind[(n, forced)]["doubled"]
    for n, forced in ((73, 1), (505, 7)):
        assert kind[(n, forced)]["chunks"] == 37 and kind[(n, forced)]["doubled"]


def test_host_batches_put_special_frames_at_every_chunk_edge():
    bank = B.encode_bank(2)
    special = [bank.index(n) for n in B.TIES]
    for n, forced in ((2048, None), (505, 7)):
        idx = B.host_idx(bank, n, forced, special, seed=1)
        start, _ = B.plan_chunks(n, forced)
        for s in start[1:-1]:
            assert idx[s - 1] in special and idx[s] in special
