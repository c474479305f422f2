"""Sweep tile configurations over the GEMM shapes of cfg1 / cfg2 (run on the GPU box). Prints us and TFLOP/s."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
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

res = []
for cfgname, (B, F, h) in {"cfg1": (4096, 1000, [512, 256, 128]), "cfg2": (8192, 2000, [1024, 512, 256])}.items():
    for name, M, N, K, amn, bmn, splits in shapes(B, F, h):
        for cg, bn in [(1, 64), (1, 128)]:
            if bn == 64 and N > 64: continue
            if bn == 256 and N <= 128: continue
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
