"""The exact CPU model of the channel pairing (DESIGN.md 7.4), and correlated test material.

Per frame: the base is the lossless model (exact_lossless: analysis, tie criterion, repair of every flagged unit of a
frame whose emitted subframes include one); a flagged unit the base does not repair (a stereo candidate that loses)
stays tied.  Every ordered pair (p, c), p != c, is the unit ch_p - ch_c analysed as any unit is (for stereo (0, 1) is
the base's difference unit as the base leaves it).  The choice is by plain enumeration of the 2^C sets of independent
channels: every other channel takes its cheapest tie-free parent in the set, the lowest between equal words; the
fewest words win, then the fewest differences, then the lexicographically smallest parent vector."""
import itertools

import numpy as np

import exact_lossless as xl
import exact_search as xs
import oracle_lib as ol

FRAME = 2048


# ----------------------------------------------------------------- choice --

def assign(I, D):
    """I[c]: words of channel c alone, None if it may not be emitted; D[p][c]: words of ch_p - ch_c, None if it may
    not -> (par tuple, words), or None where no assignment is valid."""
    C = len(I)
    best = None
    for S in range(1, 1 << C):
        members = [c for c in range(C) if S >> c & 1]
        if any(I[c] is None for c in members):
            continue
        par, total = [], 0
        for c in range(C):
            if S >> c & 1:
                par.append(c)
                total += I[c]
                continue
            opts = [(D[p][c], p) for p in members if D[p][c] is not None]
            if not opts:
                break
            w, p = min(opts)
            par.append(p)
            total += w
        else:
            key = (total, C - len(members), tuple(par))
            if best is None or key < best:
                best = key
    return None if best is None else (best[2], best[0])


def assign_brute(I, D):
    """assign() over all C^C parent vectors, by the rule as DESIGN.md 7.4 states it."""
    C = len(I)
    best = None
    for par in itertools.product(range(C), repeat=C):
        total, ok = 0, True
        for c, p in enumerate(par):
            w = I[c] if p == c else (D[p][c] if par[p] == p else None)
            if w is None:
                ok = False
                break
            total += w
        if ok:
            key = (total, sum(p != c for c, p in enumerate(par)), par)
            if best is None or key < best:
                best = key
    return None if best is None else (best[2], best[0])


# ------------------------------------------------------------------ model --

def candidate_index(C, f, p, c):
    """Where candidate (p, c) of frame f lies among the candidates' predictors: (frame, p, c) order without p = c."""
    return (f * C + p) * (C - 1) + (c if c < p else c - 1)


def model_frame(O, planes, preds=None, cand_preds=None):
    """planes: int64 [C, 2048], one frame.  preds: the base's units' predictors (order, q) or None; cand_preds:
    {(p, c): (order, q)} or None -> dict: par, emitted [(Unit, type, parent) per channel], words, base_words,
    cands {(p, c): Unit} (every pair, tied ones included; stereo (0, 1): the base's unit), tied {(p, c)}."""
    C = planes.shape[0]
    sig = list(planes) + ([planes[0] - planes[1]] if C == 2 else [])
    units = [xl.analyse(O, s) for s in sig] if preds is None else [xl.Unit(O, s, o, q) for s, (o, q) in zip(sig, preds)]
    ref = xl.emitted(units, C)
    if any(units[k].tie for k, _ in ref):
        now, stale = [xl.repair(O, u) if u.tie else u for u in units], set()
    else:
        now, stale = units, {k for k, u in enumerate(units) if u.tie}
    base_words = sum(now[k].words for k, _ in xl.emitted(now, C))
    cands, tied = {}, set()
    for p in range(C):
        for c in range(C):
            if p == c:
                continue
            if C == 2 and p == 0:
                cands[p, c] = now[2]
                if 2 in stale:
                    tied.add((p, c))
                continue
            d = planes[p] - planes[c]
            u = xl.analyse(O, d) if cand_preds is None else xl.Unit(O, d, *cand_preds[p, c])
            cands[p, c] = u
            if u.tie:
                tied.add((p, c))
    I = [None if c in stale else now[c].words for c in range(C)]
    D = [[None if p == c or (p, c) in tied else cands[p, c].words for c in range(C)] for p in range(C)]
    par, words = assign(I, D) if C > 1 else ((0,), I[0])
    em = [(now[c], 0, c) if par[c] == c else (cands[par[c], c], 1, par[c]) for c in range(C)]
    return dict(par=par, emitted=em, words=words, base_words=base_words, cands=cands, tied=tied)


def model_batch(O, pcm, channels, preds=None, frames=None):
    """-> {frame: model_frame(...)}.  preds: as selab200_encode_pairing_forced takes them ((order, q) pairs): the
    base's units first, then the candidates."""
    planes = np.asarray(pcm, np.int64).reshape(-1, FRAME, channels).transpose(0, 2, 1)
    per = 3 if channels == 2 else channels
    n_frames = planes.shape[0]
    out = {}
    for f in (range(n_frames) if frames is None else frames):
        bp = cp = None
        if preds is not None:
            bp = preds[f * per:(f + 1) * per]
            cp = {(p, c): preds[n_frames * per + candidate_index(channels, f, p, c)]
                  for p in range(channels) for c in range(channels) if p != c}
        out[f] = model_frame(O, planes[f], bp, cp)
    return out


def pack(O, model, channels):
    """The model's frames (all of a batch, in order) as (descs, words), the way the encoder lays them out."""
    descs = np.zeros(len(model) * channels, ol.DESC_DTYPE)
    words, at = [], 0
    for f in sorted(model):
        for ch, (u, t, parent) in enumerate(model[f]["emitted"]):
            kq, wq = O.rice_encode(u.q[:u.order])
            kr, wr = O.rice_encode(u.res)
            d = descs[f * channels + ch]
            d["channel"], d["subframe_type"], d["parent_channel"] = ch, t, parent
            d["refl_rice_param"], d["refl_words"], d["lpc_order"] = kq, wq.size, u.order
            d["res_rice_param"], d["res_words"], d["samples"] = kr, wr.size, FRAME
            d["refl_offset"], d["res_offset"] = at, at + wq.size
            words += [wq, wr]
            at += wq.size + wr.size
    return descs, np.concatenate(words).astype(np.uint32) if words else np.zeros(0, np.uint32)


DESC_FIELDS = ("channel", "subframe_type", "parent_channel", "refl_rice_param", "refl_words", "lpc_order",
               "res_rice_param", "res_words", "samples", "refl_offset", "res_offset")


def check_batch(O, descs, words, pcm, channels, model):
    """A whole batch equals the model's (every frame modelled): every descriptor field and every word; and it decodes
    back to its source under the port and, where built, the compiled reference."""
    md, mw = pack(O, model, channels)
    for k in DESC_FIELDS:
        assert np.array_equal(descs[k], md[k]), (k, np.nonzero(descs[k] != md[k])[0][:8])
    assert np.array_equal(words, mw)
    src = np.asarray(pcm, np.int16).reshape(-1)
    for D in [O] + ([ol.load("ref")] if ol.have_ref() else []):
        assert np.array_equal(D.decode_frames(descs, words, channels), src)


def trace_record(O, u):
    """The fields of the device's trace record of candidate unit u."""
    kq, wq = O.rice_encode(u.q[:u.order])
    kr, wr = O.rice_encode(u.res)
    c = np.zeros(xs.MAX_ORDER + 1, np.int64)
    c[1:u.order + 1] = np.asarray(u.c, np.int64)[1:u.order + 1]
    return dict(tie=int(u.tie), refl_k=kq, refl_words=wq.size, res_k=kr, res_words=wr.size, order=u.order,
                pred_digest=int(xs.pred_digest(c)), res_digest=int(xs.res_digest(np.ascontiguousarray(u.res, np.int32))))


# --------------------------------------------------------------- material --

def _clip16(x):
    return np.clip(np.rint(x), -32768, 32767).astype(np.int16)


def _source(rng, n):
    """A smooth common source: a few sines under a random walk."""
    t = np.arange(n)
    s = sum(a * np.sin(2 * np.pi * f * t + ph) for a, f, ph in
            zip(rng.uniform(1500, 6000, 4), rng.uniform(0.001, 0.05, 4), rng.uniform(0, 6.28, 4)))
    return s + np.cumsum(rng.normal(0, 30, n))


def common_source(n_frames, channels, seed, noise=20.0):
    """One source in every channel with a gain per channel near 1, plus small independent noise -> int16
    [n_frames * 2048, channels]."""
    rng = np.random.default_rng(seed)
    n = n_frames * FRAME
    s = _source(rng, n)
    gains = rng.uniform(0.8, 1.0, channels)
    return _clip16(s[:, None] * gains + rng.normal(0, noise, (n, channels)))


def dual_mono_in_six(n_frames, seed):
    """Six channels of independent noise-like material, channels 2 and 4 a dual-mono pair (equal up to +-2)."""
    rng = np.random.default_rng(seed)
    n = n_frames * FRAME
    x = np.stack([_source(rng, n) + rng.normal(0, 400, n) for _ in range(6)], axis=1)
    x[:, 4] = x[:, 2] + rng.integers(-2, 3, n)
    return _clip16(x)


def equal_and_negated(n_frames, seed):
    """Four channels: ch1 = ch0 exactly (difference all zero), ch3 = -ch2 (the difference is 2 ch2, no gain)."""
    rng = np.random.default_rng(seed)
    n = n_frames * FRAME
    a = _clip16(_source(rng, n) + rng.normal(0, 200, n)).astype(np.int64)
    b = np.clip(_clip16(_source(rng, n) + rng.normal(0, 200, n)).astype(np.int64), -32767, 32767)
    return np.stack([a, a, b, -b], axis=1).astype(np.int16)


def full_scale_opposite(n_frames, channels, seed):
    """Channels at +-full scale in opposite signs, so that differences reach +-65535."""
    rng = np.random.default_rng(seed)
    n = n_frames * FRAME
    sign = np.where(rng.integers(0, 2, (n, 1)) == 1, 1, -1)
    x = np.where(np.arange(channels)[None, :] % 2 == 0, sign * 32767 - (sign < 0), -sign * 32767 - (sign > 0))
    x = x + rng.integers(-3, 4, (n, channels)) * (np.abs(x) < 32767)
    return np.clip(x, -32768, 32767).astype(np.int16)


def families():
    """(name, pcm int16 [n, channels], channels) of small batches that exercise the pairing."""
    return (
        ("common_source_3", common_source(2, 3, 11), 3),
        ("common_source_8", common_source(2, 8, 12), 8),
        ("dual_mono_in_six", dual_mono_in_six(2, 13), 6),
        ("equal_and_negated", equal_and_negated(2, 14), 4),
        ("full_scale_opposite_2", full_scale_opposite(2, 2, 15), 2),
        ("full_scale_opposite_3", full_scale_opposite(1, 3, 16), 3),
        ("common_source_stereo", common_source(3, 2, 17), 2),
    )
