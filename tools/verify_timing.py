"""What verify costs, on BASELINE config 2/3 (44.1 kHz stereo, 10 minutes, seed 1: 12 919 frames), in one call:

  device resident   encode, decode and verify of DeviceCodec (CUDA events), and k_verify_compare on its own
                    (torch.profiler, in a pass of its own after the timed ones), its 4 B/sample read set
                    against the 3.35 TB/s of the H100 SXM data sheet;
  host buffers      selab200_encode_container against selab200_encode_container_verified (pinned buffers);
  what users do without verify
                    encode_container + container_open + container_decode + a NumPy compare per (frame, channel).

The card's name and power limit are read in the same call.
Usage: python tools/verify_timing.py [reps] [out.json]   (prints the JSON result; also writes it to out.json if named)"""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import _lib, synth  # noqa: E402
from sela_b200.device import DeviceCodec  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
OUT = sys.argv[2] if len(sys.argv) > 2 else None
HBM_BYTES_S = 3.35e12
N_FRAMES, CH, RATE = 12919, 2, 44100


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except OSError as e:
        out["power_limit_and_max_sm_clock"] = "nvidia-smi unavailable: %s" % e
    return out


def event_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def wall_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": round(statistics.median(t), 3), "min_ms": round(min(t), 3)}


def main():
    L = _lib.lib()
    _lib.init(0)
    pcm = synth.sine_noise(RATE, CH, n_frames=N_FRAMES, seed=1).reshape(-1)
    n_samples = pcm.size
    result = {"card": card(), "workload": "BASELINE config 2/3: %d frames x %d channels, %d samples" % (N_FRAMES, CH, n_samples),
              "reps": REPS}

    # ---- device resident
    dev = torch.device("cuda", 0)
    codec = DeviceCodec(N_FRAMES, CH, device=0)
    t = torch.from_numpy(pcm).to(dev)
    codec.encode(t)
    codec.check_status()
    n_words = int(codec.words_used.item())
    out = torch.empty_like(t)
    enc = event_ms(lambda: codec.encode(t), REPS)
    dec = event_ms(lambda: codec.decode(out, n_words), REPS)
    ver = event_ms(lambda: codec.verify(t, n_words), REPS)
    assert torch.equal(out, t) and codec.verify_report().size == 0
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            codec.verify(t, n_words)
        torch.cuda.synchronize()
    cmp_us = None
    for e in prof.key_averages():
        if "k_verify_compare" in e.key:
            cmp_us = getattr(e, "device_time", None) or getattr(e, "cuda_time", None)
    read = 4 * n_samples
    result["device_resident_ms"] = {
        "encode": round(enc, 3), "decode": round(dec, 3), "verify (decode + compare)": round(ver, 3),
        "k_verify_compare": round(cmp_us / 1e3, 4) if cmp_us else None}
    if cmp_us:
        result["k_verify_compare_read"] = {
            "bytes": read, "GB_s": round(read / (cmp_us * 1e-6) / 1e9, 1),
            "share_of_3.35_TB_s_data_sheet": round(read / (cmp_us * 1e-6) / HBM_BYTES_S, 3),
            "data_sheet_floor_ms": round(read / HBM_BYTES_S * 1e3, 4)}
    del codec, t, out
    torch.cuda.empty_cache()

    # ---- host buffers (pinned)
    cap = L.selab200_container_bound(N_FRAMES, CH)
    h_pcm = L.selab200_host_alloc(n_samples * 2)
    h_blob = L.selab200_host_alloc(cap)
    h_rep = L.selab200_host_alloc(N_FRAMES * CH * 16)
    h_dec = L.selab200_host_alloc(n_samples * 2)
    C.memmove(h_pcm, pcm.ctypes.data, n_samples * 2)
    used, n_rep = C.c_size_t(0), C.c_size_t(0)

    def encode():
        _lib.check(L.selab200_encode_container(h_pcm, N_FRAMES, CH, RATE, 16, h_blob, cap, C.addressof(used)))

    def encode_verified():
        _lib.check(L.selab200_encode_container_verified(h_pcm, N_FRAMES, CH, RATE, 16, h_blob, cap, C.addressof(used),
                                                        h_rep, N_FRAMES * CH, C.addressof(n_rep)))

    src = pcm.reshape(N_FRAMES, 2048, CH)
    decoded = np.ctypeslib.as_array(C.cast(h_dec, C.POINTER(C.c_int16)), shape=(n_samples,))

    def today():  # what a user has to do without verify: encode, read the bytes back, compare in NumPy
        encode()
        info = np.zeros(1, _lib.INFO_DTYPE)
        h = C.c_void_p(0)
        _lib.check(L.selab200_container_open(h_blob, used.value, C.addressof(h), info.ctypes.data))
        try:
            _lib.check(L.selab200_container_decode(h, h_dec))
        finally:
            L.selab200_container_close(h)
        bad = (decoded.reshape(N_FRAMES, 2048, CH) != src).any(axis=1)
        return np.argwhere(bad)

    rows = []
    for _ in range(3):   # alternated, so that drift on a shared host hits all three alike
        rows.append((wall_ms(encode, REPS // 2), wall_ms(encode_verified, REPS // 2), wall_ms(today, REPS // 4)))
    blob_verified = bytes(C.string_at(h_blob, used.value))
    encode()
    assert bytes(C.string_at(h_blob, used.value)) == blob_verified and n_rep.value == 0 and today().size == 0
    pick = lambda i: min(r[i]["median_ms"] for r in rows)  # noqa: E731
    result["host_buffers_ms (best of 3 alternated medians)"] = {
        "encode_container": pick(0), "encode_container_verified": pick(1),
        "encode_container + container_open + container_decode + NumPy compare": pick(2),
        "verify share of encode_container_verified": round(1 - pick(0) / pick(1), 3)}
    result["host_buffers_runs"] = rows
    for p in (h_pcm, h_blob, h_rep, h_dec):
        L.selab200_host_free(p)

    if OUT:
        with open(OUT, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
