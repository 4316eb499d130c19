"""The exact CPU model of the search + pairing (DESIGN.md 7.5), built on the models of its two parts.

Per frame: the base is the order search (exact_search.model_batch_all: every analysis unit at its searched order); no
searched unit has a tie, so none is stale.  Every ordered pair (p, c), p != c, is the unit ch_p - ch_c with all 100 q of
its own analysis (exact_search.all_q of the difference signal) searched over orders 1..100 as any unit is
(exact_search.search_units); for stereo (0, 1) is the base's searched difference unit.  The choice is
exact_pairing.assign on the searched words, and the stream is laid out as exact_pairing.pack lays it out."""
import numpy as np

import exact_pairing as xp
import exact_search as xs

FRAME = 2048
MAX_ORDER = xs.MAX_ORDER


def candidates(channels):
    """The candidates (p, c) that are sized, in (p, c) order: p != c, and for stereo only (1, 0)."""
    return [(p, c) for p in range(channels) for c in range(channels) if p != c and not (channels == 2 and p == 0)]


def _coded(m, Q, u):
    o = int(m["order"][u])
    return xs.Coded(o, np.where(np.arange(MAX_ORDER) < o, Q[u], 0).astype(np.int32), m["res"][u],
                    int(m["words"][u, o - 1]))


def model_batch(pcm, channels, preds=None):
    """-> (model, cand, index, Qc, refc) for every frame of a batch.

    model {frame: dict(par, emitted [(Coded, type, parent) per channel], words, base_words, cands {(p, c): Coded},
    I, D)}; cand: search_units' dict of the candidates, one row per sized candidate; index {(frame, p, c): row};
    Qc, refc: the candidates' q and reference orders.  preds: (order, q[100]) pairs as
    selab200_encode_search_pairing_forced takes them: the base's units, then every candidate (frame, p, c), p != c."""
    planes = np.asarray(pcm, np.int64).reshape(-1, FRAME, channels).transpose(0, 2, 1)
    n_frames, per = planes.shape[0], 3 if channels == 2 else channels
    n_units = n_frames * per
    base_preds = None if preds is None else preds[:n_units]
    base, _, m, Q, _ = xs.model_batch_all(pcm, channels, base_preds)
    pairs = candidates(channels)
    index = {(f, p, c): i for i, (f, (p, c)) in enumerate((f, pc) for f in range(n_frames) for pc in pairs)}
    S = np.array([planes[f, p] - planes[f, c] for f, p, c in index], np.int64).reshape(-1, FRAME)
    if preds is None:
        Qc, refc = xs.all_q(S) if S.shape[0] else (np.zeros((0, MAX_ORDER), np.int32), np.zeros(0, int))
    else:
        rows = [preds[n_units + xp.candidate_index(channels, f, p, c)] for f, p, c in index]
        Qc = np.array([np.asarray(q, np.int32)[:MAX_ORDER] for _, q in rows], np.int32).reshape(-1, MAX_ORDER)
        refc = np.array([int(o) for o, _ in rows], int)
    mc = xs.search_units(S, Qc, refc) if S.shape[0] else None
    out = {}
    for f in range(n_frames):
        units = [_coded(m, Q, f * per + k) for k in range(per)]
        cands = {(p, c): _coded(mc, Qc, index[f, p, c]) for p, c in pairs}
        if channels == 2:
            cands[0, 1] = units[2]
        I = [units[c].words for c in range(channels)]
        D = [[None if p == c else cands[p, c].words for c in range(channels)] for p in range(channels)]
        par, words = xp.assign(I, D) if channels > 1 else ((0,), I[0])
        em = [(units[c], 0, c) if par[c] == c else (cands[par[c], c], 1, par[c]) for c in range(channels)]
        base_words = sum(u.words for u, _ in base[f])
        out[f] = dict(par=par, emitted=em, words=words, base_words=base_words, cands=cands, I=I, D=D)
    return out, mc, index, Qc, refc


def pack(O, model, channels):
    """The model's frames (all of a batch, in order) as (descs, words), the way the encoder lays them out."""
    return xp.pack(O, model, channels)


def check_batch(O, descs, words, pcm, channels, model):
    """A whole batch equals the model's, every descriptor field and every word, and decodes back to its source under
    the port and, where built, the compiled reference."""
    xp.check_batch(O, descs, words, pcm, channels, model)
