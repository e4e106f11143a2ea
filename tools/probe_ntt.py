"""GPU probe: time our NTT (device-resident) against the reference's own kernels built for
sm_90a (oracle/_ref), over the kernel variants selected by environment knobs.  Two clocks per
case: `call` = one call between two events (includes the host-side launch path while the GPU is
idle), `b2b` = 20 calls back to back divided by 20 (the GPU never waits for the host: kernel time).
Development tool, not the bench."""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sppark_b200 import ntt, _lib  # noqa: E402

GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001


def time_fn(fn, stream, iters=10, warm=3, flush=None, batch=20):
    for _ in range(warm):
        fn()
    stream.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1)
            torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    bs = []
    for _ in range(3):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(batch):
            fn()
        e1.record(stream)
        e1.synchronize()
        bs.append(e0.elapsed_time(e1) / batch)
    return ts[len(ts) // 2], min(bs)


KNOBS = ["SPPARK_B200_NTT_CPT", "SPPARK_B200_NTT_BLOCK", "SPPARK_B200_NTT_SPLIT"]


def main():
    torch.cuda.init()
    print(torch.cuda.get_device_name(0))
    cur = torch.cuda.current_stream()
    flush = torch.zeros(64 << 20, dtype=torch.int32, device="cuda")      # 256 MiB > L2
    args = sys.argv[1:]
    fields = ["gl64"]
    if args and args[0] in ("gl64", "bb31", "both", "bls12_381"):
        if args[0] == "both":
            # one reference library per process (their parameter statics are STB_GNU_UNIQUE symbols)
            import subprocess
            for f in ("gl64", "bb31"):
                subprocess.check_call([sys.executable, os.path.abspath(__file__), f] + args[1:])
            return
        fields = [args[0]]
        args = args[1:]
    sizes = [int(a) for a in args] or [16, 20, 22, 24]
    l = _lib.lib()
    for field in fields:
        for lg in sizes:
            n = 1 << lg
            rng = np.random.default_rng(lg)
            if field == "gl64":
                host = rng.integers(0, GL_P, size=n, dtype=np.uint64)
                view, fid, esz = np.int64, 0, 8
            elif field == "bb31":
                host = rng.integers(0, BB_P, size=n, dtype=np.uint32)
                view, fid, esz = np.int32, 1, 4
            else:
                host = rng.integers(0, 2**62, size=(n, 4), dtype=np.uint64)      # valid residues of BLS12-381 fr
                view, fid, esz = np.int64, 2, 32
            bytes_alg = 2 * n * esz
            variants = [("warp", {}), ("block", {"SPPARK_B200_NTT_BLOCK": "1"})]
            if lg == 20:
                variants += [("warp 7,7,6", {"SPPARK_B200_NTT_SPLIT": "7,7,6"})]
            for vname, env in variants:
                for k in KNOBS:
                    os.environ.pop(k, None)
                os.environ.update(env)
                for order, name in ((ntt.NN, "NN"), (ntt.NR, "NR"), (ntt.RN, "RN")):
                    d = torch.from_numpy(host.view(view)).cuda()
                    ptr, s = d.data_ptr(), cur.cuda_stream
                    med, b2b = time_fn(lambda: l.sppark_b200_ntt_dev(fid, ptr, lg, order, 0, 0, s), cur,
                                       flush=flush if lg >= 22 else None)
                    print(f"ours[{vname}] {field} 2^{lg} {name}: call {med*1e3:.1f} us  b2b {b2b*1e3:.1f} us  "
                          f"-> {bytes_alg/ (b2b*1e-3) / 1e9:.0f} GB/s algorithmic", flush=True)
            for k in KNOBS:
                os.environ.pop(k, None)
            # reference kernels, same box, data resident
            p = os.path.join(ROOT, "oracle", "_ref", f"libref_ntt_{field}_gpu.so")
            if os.path.exists(p):
                ref = C.CDLL(p)
                ref.ref_ntt_stream.restype = C.c_void_p
                ref.ref_ntt_dev_async.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int]
                rs = torch.cuda.ExternalStream(ref.ref_ntt_stream())
                for order, name in ((0, "NN"), (1, "NR"), (2, "RN")):
                    d = torch.from_numpy(host.view(view)).cuda()
                    torch.cuda.synchronize()
                    ptr = d.data_ptr()
                    med, b2b = time_fn(lambda: ref.ref_ntt_dev_async(ptr, lg, order, 0, 0), rs,
                                       flush=flush if lg >= 22 else None)
                    print(f"REF   {field} 2^{lg} {name}: call {med*1e3:.1f} us  b2b {b2b*1e3:.1f} us  "
                          f"-> {bytes_alg/ (b2b*1e-3) / 1e9:.0f} GB/s algorithmic", flush=True)
                if field == "gl64":
                    d1 = torch.from_numpy(host.view(view)).cuda()
                    d2 = d1.clone()
                    ntt.ntt_dev(d1, ntt.NN)
                    torch.cuda.synchronize()
                    ref.ref_ntt_dev_async(d2.data_ptr(), lg, 0, 0, 0)
                    rs.synchronize()
                    print(f"ours == reference-GPU at 2^{lg} NN:", bool(torch.equal(d1, d2)), flush=True)
    print("launches:", _lib.launch_count())


if __name__ == "__main__":
    main()
