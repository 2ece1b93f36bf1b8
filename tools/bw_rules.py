"""Bandwidth shape of the HBM-bound kernels of the path (SURVEY 8d): plane encoding and legal-move generation on 65,536
positions (seeded random playouts, plies 0-80, all of one variant), achieved GB/s against the measured HBM peak.

  python tools/bw_rules.py [variant_id mode version]        (defaults: crazyhouse 1 0 1)
  ncu --set full -k regex:'encode_planes|legal_moves' -c 4 ... python tools/bw_rules.py    (profiles/r02_ncu_rules_kernels.json)
"""
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N = 65536


def positions(variant, n, seed=42):
    from crazyara_b200.engine import BoardState
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        st = BoardState().set("", False, variant)
        plies = int(rng.integers(0, 81))
        for _ in range(plies):
            mv = st.legal_actions()
            if not mv or st.is_terminal() != 4:
                break
            st.do_action(mv[int(rng.integers(len(mv)))])
            out.append(st.board())
            if len(out) >= n:
                break
        out.append(st.board())
    return out[:n]


def main():
    import torch
    from crazyara_b200 import lib
    from crazyara_b200.engine import AraBoard, legal_moves_gpu, planes_channels
    variant, mode, version = (int(x) for x in (sys.argv[1:4] if len(sys.argv) >= 4 else (1, 0, 1)))
    channels = planes_channels(mode, version)
    t0 = time.time()
    boards = positions(variant, N)
    arr = (AraBoard * N)(*boards)
    host = np.frombuffer(arr, dtype=np.uint8).reshape(N, 128)
    d_boards = torch.from_numpy(host.copy()).cuda()
    L = lib()
    L.ara_encode_planes_device.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    d_f32 = torch.empty((N, channels, 8, 8), dtype=torch.float32, device="cuda")
    cpad = 64 if channels <= 64 else 128
    d_f16 = torch.empty((N, 64, cpad), dtype=torch.float16, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 6500.0))
    out = {"positions": N, "variant": variant, "mode": mode, "version": version, "channels": channels, "hbm_peak_gbs": peak,
           "generation_s": round(time.time() - t0, 1)}

    def timed(fn, reps=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
        ev[0].record()
        for i in range(reps):
            fn()
            ev[i + 1].record()
        torch.cuda.synchronize()
        return min(ev[i].elapsed_time(ev[i + 1]) for i in range(reps)) * 1e-3

    s = timed(lambda: L.ara_encode_planes_device(d_boards.data_ptr(), N, mode, version, 1, d_f32.data_ptr(), None, 0, stream))
    b = N * (channels * 64 * 4 + 128)
    out["encode_planes_f32"] = {"seconds": s, "algorithmic_bytes": b, "gbs": b / s / 1e9, "frac_of_hbm_peak": b / s / 1e9 / peak,
                                "bytes_per_position": channels * 64 * 4 + 128}
    s = timed(lambda: L.ara_encode_planes_device(d_boards.data_ptr(), N, mode, version, 1, None, d_f16.data_ptr(), cpad, stream))
    b = N * (64 * cpad * 2 + 128)
    out["encode_planes_f16_nhwc"] = {"seconds": s, "algorithmic_bytes": b, "gbs": b / s / 1e9, "frac_of_hbm_peak": b / s / 1e9 / peak,
                                     "bytes_per_position": 64 * cpad * 2 + 128}
    # legal moves: host-buffer entry (the kernel's own duration comes from the ncu capture); moves written: 2 B per move
    t1 = time.perf_counter()
    moves, term, pidx = legal_moves_gpu(boards)
    wall = time.perf_counter() - t1
    n_moves = sum(len(m) for m in moves)
    out["legal_moves"] = {"host_call_seconds": wall, "moves_generated": n_moves, "mean_moves": n_moves / N,
                          "algorithmic_bytes": N * (128 + 4 + 4) + n_moves * (2 + 4),
                          "note": "ara_legal_moves with host buffers (H2D boards, kernel, D2H moves/indices); kernel time: ncu capture"}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
