import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["SB_GEMM_TRACE"] = "1"
import shifu_tensorflow_b200 as sb
B = 4096
for (M, N, K, amn, bmn, cg, bn, sk) in [(B, 128, 256, False, True, 1, 128, 1), (B, 512, 1000, False, True, 1, 128, 1),
                                         (B, 256, 128, False, False, 1, 128, 1), (256, 128, B, True, True, 1, 128, 8),
                                         (8192, 1024, 2000, False, True, 1, 128, 1)]:
    ms = sb.capi.debug_gemm_bench(M, N, K, split_k=sk, a_mn=amn, b_mn=bmn, cg=cg, bn=bn, iters=20)
    print("avg back-to-back %.2f us" % (ms * 1e3), flush=True)
