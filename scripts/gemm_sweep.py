"""Sweep tile configurations over the GEMM shapes of cfg1 / cfg2 (run on the GPU box). Prints us and TFLOP/s.
Forward and dA GEMMs run with their real epilogues (relu): on the ping-pong kernel once per warpgroup tile height
(bm_wg 64 / 128), forward GEMMs also on the 128 x 256 tile of gemm_wide.cuh (bm_wg 256); "plan" marks the planner's
choice.  dW GEMMs (gemm_dw.cuh) over tile width (64 / 128 / 256) and split-K."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import shifu_tensorflow_b200 as sb

def shapes(B, F, h):
    dims = [F] + h
    out = []
    for l in range(len(h)):
        out.append(("fwd%d" % (l + 1), B, dims[l + 1], dims[l], False, True, [1]))
    for l in range(len(h) - 1, -1, -1):
        out.append(("dW%d" % (l + 1), dims[l], dims[l + 1], B, True, True, [1, 2, 4, 8, 16]))
        if l > 0:
            out.append(("dA%d" % (l + 1), B, dims[l], dims[l + 1], False, False, [1]))
    return out

def planned_bm_wg(M, N, K, fwd, sms=132):   # plan_gemm_pp (gemm_pp.cuh)
    tm, kb = (M + 127) // 128, (K + 63) // 64
    wide, narrow = tm * ((N + 255) // 256), tm * ((N + 127) // 128)
    if fwd and N > 128 and 8 * wide >= 7 * sms and kb >= 16 and 2 * -(-wide // sms) <= -(-narrow // sms):
        return 256
    bn = 64 if N <= 64 else 128
    t = tm * ((N + bn - 1) // bn)
    return 128 if t > sms or (8 * t >= 7 * sms and kb >= 8) else 64

res = []
rng = np.random.default_rng(0)
for cfgname, (B, F, h) in {"cfg1": (4096, 1000, [512, 256, 128]), "cfg2": (8192, 2000, [1024, 512, 256])}.items():
    for name, M, N, K, amn, bmn, splits in shapes(B, F, h):
        if not amn:   # forward / dA: the ping-pong kernel
            da = not bmn
            A = rng.standard_normal((M, K), dtype=np.float32)
            W = rng.standard_normal((N, K) if da else (K, N), dtype=np.float32)
            kw = dict(aux=rng.uniform(0, 1, (M, N)).astype(np.float32)) if da else dict(bias=np.zeros(N, np.float32))
            for bm in (64, 128) if da else (64, 128, 256):
                _, _, ms = sb.capi.debug_gemm_epilogue(A, W, sb.capi.ACT_RELU, bm_wg=bm, iters=30, **kw)
                tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
                tag = "plan" if bm == planned_bm_wg(M, N, K, not da) else ""
                print("%s %-5s M=%5d N=%5d K=%5d bm_wg=%3d  %8.2f us  %7.1f TF %s" % (cfgname, name, M, N, K, bm, ms * 1e3, tf, tag), flush=True)
                res.append(dict(cfg=cfgname, name=name, M=M, N=N, K=K, bm_wg=bm, us=ms * 1e3, tflops=tf))
            continue
        for cg, bn in [(1, 64), (1, 128), (1, 256)]:
            if (bn == 64 and N > 64) or (bn == 256 and N <= 128): continue
            for sk in splits:
                try:
                    ms = sb.capi.debug_gemm_bench(M, N, K, split_k=sk, a_mn=amn, b_mn=bmn, cg=cg, bn=bn, iters=30)
                except Exception as e:
                    print(cfgname, name, cg, bn, sk, "ERR", e); continue
                tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
                print("%s %-5s M=%5d N=%5d K=%5d cg=%d bn=%3d split=%2d  %8.2f us  %7.1f TF" % (cfgname, name, M, N, K, cg, bn, sk, ms * 1e3, tf), flush=True)
                res.append(dict(cfg=cfgname, name=name, M=M, N=N, K=K, cg=cg, bn=bn, split=sk, us=ms * 1e3, tflops=tf))
if len(sys.argv) > 1:       # optional: the sweep as JSON, to the path given
    json.dump(res, open(sys.argv[1], "w"))
