"""Developer tool: validate the MN-major wgmma operand path of sb_gemm_bf16_tn against torch.

Sweeps the descriptor-field candidates (LBO, SBO, K advance) so that one GPU call settles the
encoding; the defaults compiled into gemm.cu are the first row."""
import sys
import torch
sys.path.insert(0, ".")
from speech_b200 import _lib, ops
lib = _lib.load()
torch.manual_seed(0)
cands = [(8192, 1024, 2048), (1024, 8192, 2048), (8192, 1024, 256), (8192, 128, 2048),
         (128, 1024, 2048)]
shapes = [(128, 64, 256), (256, 128, 192), (384, 256, 512), (512, 512, 2048), (300, 200, 1000),
          (3072, 2048, 4096)]
for lbo, sbo, kadv in cands:
    lib.sb_debug_umma_mn(lbo, sbo, kadv)
    worst = {}
    for (M, N, K) in shapes:
        A = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        B = torch.randn(N, K, device="cuda").to(torch.bfloat16)
        ref = A.float() @ B.float().t()
        Mp, Np = (M + 7) // 8 * 8, (N + 7) // 8 * 8
        At = torch.zeros(K, Mp, device="cuda", dtype=torch.bfloat16); At[:, :M] = A.t()
        Bt = torch.zeros(K, Np, device="cuda", dtype=torch.bfloat16); Bt[:, :N] = B.t()
        for name, (a, b, am, bm) in {"a_mn": (At[:, :M], B, True, False),
                                     "b_mn": (A, Bt[:, :N], False, True),
                                     "ab_mn": (At[:, :M], Bt[:, :N], True, True)}.items():
            for acc in (False, True):
                try:
                    if acc:
                        out = torch.zeros(M, N, device="cuda")
                        ops.gemm_bf16_tn(a, b, out=out, accumulate=True, split_k=2, a_mn=am, b_mn=bm)
                    else:
                        out = ops.gemm_bf16_tn(a, b, a_mn=am, b_mn=bm)
                    torch.cuda.synchronize()
                    err = ((out - ref).abs().max() / ref.abs().max()).item()
                except Exception as e:
                    err = float("nan")
                    print("   error", name, (M, N, K), repr(e)[:100])
                worst[name] = max(worst.get(name, 0.0), err if err == err else 9e9)
    print("lbo %5d sbo %5d kadv %5d :" % (lbo, sbo, kadv),
          "  ".join("%s %.2e" % kv for kv in worst.items()), flush=True)
lib.sb_debug_umma_mn(8192, 1024, 2048)
