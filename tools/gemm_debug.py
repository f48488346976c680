"""Diagnostics for the wgmma GEMM (run on the GPU box when a test_gemm case fails): per-layout error statistics and
a k-slice probe (A non-zero only in one 16-wide k-step) that localises descriptor / swizzle mistakes."""
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from pytorch_distributed_nlp_b200 import _lib as L

dev = torch.device("cuda", 0)


def call(M, N, K, A, lda, am, B, ldb, bm, D, bn=0, splits=0, ws=None):
    a = L.GemmArgs()
    a.M, a.N, a.K = M, N, K
    a.A, a.lda, a.a_major = A.data_ptr(), lda, am
    a.B, a.ldb, a.b_major = B.data_ptr(), ldb, bm
    a.D, a.ldd, a.epilogue = D.data_ptr(), N, 0
    a.force_bn, a.force_splits = bn, splits
    a.workspace, a.workspace_bytes = (ws.data_ptr() if ws is not None else None), (ws.numel() if ws is not None else 0)
    try:
        L.call("b2_gemm_bf16", a, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return True
    except Exception as e:  # noqa
        print("   EXC", str(e)[:300])
        return False


def stats(tag, D, ref):
    err = (D.float() - ref).abs()
    scale = ref.abs().max().item() + 1e-9
    bad = err > 0.02 * scale
    msg = "%-44s max_err %.4g scale %.4g bad %.4f%%" % (tag, err.max().item(), scale, 100 * bad.float().mean().item())
    if bad.any():
        idx = bad.nonzero()[:6].tolist()
        rows = bad.any(1).nonzero().flatten()
        cols = bad.any(0).nonzero().flatten()
        msg += "  first bad %s rows[%d..%d] n=%d cols[%d..%d] n=%d" % (
            idx, rows.min().item(), rows.max().item(), rows.numel(), cols.min().item(), cols.max().item(), cols.numel())
    print(msg, flush=True)
    return not bad.any()


def main():
    torch.manual_seed(0)
    for (name, am, bm) in (("NT", 0, 0), ("NN", 0, 1), ("TN", 1, 1)):
        for bn in (128, 192, 256):
            M, N, K = 256, 768, 128
            A = torch.randn(M, K, device=dev).to(torch.bfloat16)
            Bt = (torch.randn(N, K, device=dev) * 0.1).to(torch.bfloat16)
            ref = A.float() @ Bt.float().t()
            Aop = A if am == 0 else A.t().contiguous()          # MN-major: stored [K, M]
            Bop = Bt if bm == 0 else Bt.t().contiguous()        # MN-major: stored [K, N]
            lda = K if am == 0 else M
            ldb = K if bm == 0 else N
            D = torch.zeros(M, N, dtype=torch.bfloat16, device=dev)
            if not call(M, N, K, Aop, lda, am, Bop, ldb, bm, D, bn=bn):
                return
            ok = stats("%s bn=%d M%d N%d K%d" % (name, bn, M, N, K), D, ref)
            if not ok:
                for ks in range(K // 16):
                    A2 = torch.zeros_like(A)
                    A2[:, ks * 16:(ks + 1) * 16] = A[:, ks * 16:(ks + 1) * 16]
                    Aop2 = A2 if am == 0 else A2.t().contiguous()
                    D.zero_()
                    call(M, N, K, Aop2, lda, am, Bop, ldb, bm, D, bn=bn)
                    stats("   k-step %d only" % ks, D, A2.float() @ Bt.float().t())


if __name__ == "__main__":
    main()
