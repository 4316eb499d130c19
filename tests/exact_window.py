"""The exact CPU model of the window search (DESIGN.md 7.6), built on exact_analysis and exact_search.

Per analysis unit: the base is the order search (exact_search.model_batch_all), its winner's words S.  For every
selected window w the unit's signal is analysed as exact_analysis.analyse analyses it, except that the mean-removed
signal is multiplied by the window first -- d = x - mean, then d * w, one rounded multiply, then one sequential chain
per lag in the same order -- and all 100 q of that analysis are searched over orders 1..100 with no reference order
(exact_search.search_units), each q clamped to [-64, 63] first (window_q); an order whose predictor leaves the domain
of the int64 conversion counts as tied (_search_records).  The unit takes the tie-free window candidate with the fewest words if that is strictly
fewer than S, between equal words the lower window, then the lower order; otherwise it keeps the order search's winner.
The stereo decision then runs on the chosen units.  numpy's float64 operations are IEEE-rounded and never fused, so the
model is bitwise exact.  The windows are inputs: the tests read the encoder's table through
sela_b200.codec.analysis_window, so that model and encoder multiply by the same doubles."""
import numpy as np

import analysis_corpus
import exact_analysis as xa
import exact_search as xs

FRAME = 2048
MAX_ORDER = xs.MAX_ORDER
N_WINDOWS = 5


def mask_rows(mask):
    """The table rows a window mask selects, in increasing bit order."""
    return [i for i in range(N_WINDOWS) if mask >> i & 1]


def analyse_windowed(s, w):
    """s: int [F, N] signals, w: float64 [N] -> dict of mean[F], ac[F, 101] (normalised), k[F, 100] and q[F, 100]
    (every coefficient quantised; no order is chosen)."""
    s = np.atleast_2d(np.asarray(s, np.int64))
    w = np.asarray(w, np.float64)
    F, N = s.shape
    x = s.astype(np.float64) / 32767.0
    total = np.zeros(F)
    for j in range(N):
        total = total + x[:, j]
    mean = total / N
    d = (x - mean[:, None]) * w[None, :]
    ac = np.zeros((F, xa.LAGS))
    for j in range(N):
        m = min(j, xa.LAGS - 1)
        ac[:, :m + 1] = ac[:, :m + 1] + d[:, j:j + 1] * d[:, j - m:j + 1][:, ::-1]
    with np.errstate(invalid="ignore", divide="ignore"):
        ac[:, 1:] = ac[:, 1:] / ac[:, :1]                    # a window that sees only silence: NaN, then q = 0
        ac[:, 0] = 1.0
        g0 = ac[:, 1:].copy()
        g1 = g0.copy()
        err = ac[:, 0].copy()
        k = np.zeros((F, MAX_ORDER))
        for i in range(MAX_ORDER):
            if i:
                kp = k[:, i - 1:i]
                n = MAX_ORDER - i
                up = g1[:, 1:n + 1].copy()
                g1[:, :n] = up + kp * g0[:, :n]
                g0[:, :n] = up * kp + g0[:, :n]
            head = g1[:, 0]
            k[:, i] = -head / err
            err = err + head * k[:, i]
    q0, q1, qr = xa.quantise(k)
    q = qr.copy()
    q[:, 0] = q0[:, 0]
    q[:, 1] = q1[:, 1]
    return dict(mean=mean, ac=ac, k=k, q=q)


def quantise_clamped(k):
    """k float64 [F, 100] -> the q a window record holds (int32): each coefficient through quantizeReflectionCoefficients'
    formula (exact_analysis.quantise), NaN to 0, and clamped to [-64, 63] while still a double, as the device clamps
    the quantiser's saturating conversion; an infinite or huge k gives 63 or -64, not a wrapped integer."""
    k = np.asarray(k, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        v = np.floor(64.0 * k)
        v[:, 0] = np.floor(64.0 * (-1.0 + xa.SQRT2 * np.sqrt(k[:, 0] + 1.0)))
        v[:, 1] = np.floor(64.0 * (-1.0 + xa.SQRT2 * np.sqrt(-k[:, 1] + 1.0)))
    return np.where(np.isnan(v), 0.0, np.clip(v, -64.0, 63.0)).astype(np.int32)


def window_q(s, w):
    """The q a window record holds: every q of the windowed analysis, clamped to [-64, 63], the range the decoders
    read.  A near-singular windowed analysis can round to |k| > 1, which the quantiser maps outside it."""
    return quantise_clamped(analyse_windowed(s, w)["k"])


def choose(base_words, rec_words, rec_order):
    """The rule of 7.6 for one unit: base_words its order search winner's words, rec_words[w] and rec_order[w] each
    window record's best (fewest words, then lowest order) -> (window or None, order, words)."""
    key = min((int(wd), w, int(o)) for w, (wd, o) in enumerate(zip(rec_words, rec_order)))
    return (key[1], key[2], key[0]) if key[0] < base_words else (None, None, int(base_words))


def _search_records(S, Q):
    """exact_search.search_units on window records (no reference order), with every order whose predictor leaves the
    domain of the int64 conversion counted as tied: never eligible.  The records whose winner that moves get the new
    winner's order, key and residues."""
    mw = xs.search_units(S, Q, np.zeros(S.shape[0], int))
    out = ~mw["domain"]
    if not out.any():
        return mw
    mw["tie"] = mw["tie"] | out
    orders = np.arange(1, MAX_ORDER + 1)
    key = np.where(mw["tie"], np.iinfo(np.int64).max, mw["words"] * 256 + orders)
    win = np.argmin(key, axis=1)
    for r in np.flatnonzero(win + 1 != mw["order"]):
        C, _ = xs.predictors_all(Q[r:r + 1])
        res, _ = xs.fir_limbs(S[r:r + 1], C)
        mw["res"][r] = res[0, win[r]]
    mw["best"] = key[np.arange(key.shape[0]), win]
    mw["order"] = win + 1
    return mw


def model_batch(pcm, channels, tables, preds=None):
    """-> (model, base_words, mw, Qw, chosen) for every frame of a batch with the windows `tables` (float64 [n, 2048]).

    model {frame: [(Coded, type) per channel]} as exact_search lays it out; base_words {frame: the order search's
    words}; mw: search_units' dict of the (unit, window) records, row unit * n + w, and in mw["unit_keys"] every
    unit's window key words << 16 | w << 8 | order; Qw int32 [n_units, n, 100];
    chosen[u]: the window a unit is coded from, or -1.  preds: (order, q[100]) pairs as
    selab200_encode_search_windows_forced takes them (the units', then the records')."""
    tables = np.atleast_2d(np.asarray(tables, np.float64))
    n = tables.shape[0]
    S = analysis_corpus.units(pcm, channels)
    per = 3 if channels == 2 else channels
    U = S.shape[0]
    base, _, m, Q, _ = xs.model_batch_all(pcm, channels, None if preds is None else preds[:U])
    if preds is None:
        Qw = np.stack([window_q(S, t) for t in tables], axis=1) if U else np.zeros((0, n, MAX_ORDER))
    else:
        Qw = np.array([np.asarray(q, np.int32)[:MAX_ORDER] for _, q in preds[U:]]).reshape(U, n, MAX_ORDER)
    Qw = np.asarray(Qw, np.int32).reshape(U, n, MAX_ORDER)
    mw = _search_records(np.repeat(S, n, axis=0), Qw.reshape(-1, MAX_ORDER))
    rec_words = (mw["best"] >> 8).reshape(U, n)
    rec_order = mw["order"].reshape(U, n)
    mw["unit_keys"] = ((rec_words << 16) | (np.arange(n)[None, :] << 8) | rec_order).min(axis=1).astype(np.uint64)
    chosen = np.full(U, -1)
    units = []
    for u in range(U):
        w, o, words = choose(int(m["best"][u] >> 8), rec_words[u], rec_order[u])
        if w is None:
            o = int(m["order"][u])
            units.append(xs.Coded(o, np.where(np.arange(MAX_ORDER) < o, Q[u], 0).astype(np.int32), m["res"][u],
                                  int(m["words"][u, o - 1])))
        else:
            chosen[u] = w
            units.append(xs.Coded(o, np.where(np.arange(MAX_ORDER) < o, Qw[u, w], 0).astype(np.int32),
                                  mw["res"][u * n + w], words))
    model, base_words = {}, {}
    for f in range(U // per):
        fu = units[f * per:(f + 1) * per]
        model[f] = [(fu[k], t) for k, t in xs.emitted(fu, channels)]
        base_words[f] = sum(c.words for c, _ in base[f])
    return model, base_words, mw, Qw, chosen


def music_like(n_frames, channels, seed):
    """Coloured test audio, int16 [n_frames * 2048, channels]: per channel a few decaying harmonics of a note that
    changes every frame, plus AR(8)-coloured noise.  Deterministic."""
    rng = np.random.default_rng(seed)
    n = n_frames * FRAME
    t = np.arange(n, dtype=np.float64)
    ar = np.array([1.8, -1.3, 0.6, -0.2, 0.1, -0.05, 0.02, -0.01])
    out = np.zeros((n, channels))
    for c in range(channels):
        for f in range(n_frames):
            sl = slice(f * FRAME, (f + 1) * FRAME)
            f0 = rng.uniform(0.005, 0.08)
            env = np.exp(-np.arange(FRAME) / rng.uniform(300, 3000))
            for h in range(1, 6):
                out[sl, c] += rng.uniform(500, 6000) / h * env * np.sin(f0 * h * t[sl] + rng.uniform(0, 6.3))
        e = rng.standard_normal(n) * rng.uniform(20, 300)
        a = np.zeros(n + 8)
        for j in range(n):
            a[j + 8] = e[j] + ar @ a[j:j + 8][::-1]
        out[:, c] += a[8:]
    return np.clip(np.rint(out), -32768, 32767).astype(np.int16)


def pack(O, model, channels):
    return xs.pack(O, model, channels)


def check_frames(O, descs, words, pcm, channels, model):
    xs.check_frames(O, descs, words, pcm, channels, model)
