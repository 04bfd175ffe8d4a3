"""GPU: wgmma descriptor conventions (avc_tc_probe_gemm) -- the foundation of the tensor-core
conv kernels.  TF32 inputs (10-bit mantissa, truncated by the tensor core), fp32 accumulate:
tolerance 2e-3 of max."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def img_kmajor(mat, rows_total=None, row0=0):
    """[R][K] matrix -> image [K/4][rows_total][4] (the A4 / packed-weight smem layout)."""
    R, K = mat.shape
    rows_total = rows_total or R
    img = torch.zeros(K // 4, rows_total, 4)
    img[:, row0:row0 + R] = mat.reshape(R, K // 4, 4).permute(1, 0, 2)
    return img.contiguous()


def run_probe(a_img, b_img, strides, nk, N, a_mn=0, b_mn=0, reps=1, want_cycles=False):
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    a, b = a_img.cuda().contiguous(), b_img.cuda().contiguous()
    D = torch.full((128, N), float("nan"), device="cuda")
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    strides = list(strides) + [0] * (10 - len(strides))
    st = (C.c_uint32 * 10)(*strides)
    L.check(lib.avc_tc_probe_gemm(a.data_ptr(), a.numel() * 4, b.data_ptr(), b.numel() * 4, st, nk, N, a_mn, b_mn, reps,
                                  D.data_ptr(), status.data_ptr(), torch.cuda.current_stream().cuda_stream), "probe")
    torch.cuda.synchronize()
    assert int(status[0]) == 0, "probe reported a failure"
    if want_cycles:
        return D.cpu(), int(status[1])
    return D.cpu()


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("N,K", [(128, 16), (256, 64), (144, 32), (16, 8)])
def test_kmajor_gemm(N, K):
    g = torch.Generator().manual_seed(N + K)
    A, B = torch.randn((128, K), generator=g), torch.randn((N, K), generator=g)
    strides = [128 * 16, 128, N * 16, 128, 2 * 128 * 16, 2 * N * 16, 0, 0]
    D = run_probe(img_kmajor(A), img_kmajor(B), strides, K // 8, N)
    assert rel(D, A @ B.t()) < 2e-3, rel(D, A @ B.t())


def test_row_offset_is_a_tap_shift():
    """B rows [j, j+N) of a taller image: descriptor start + j*16 bytes (how the 5 conv taps
    address one staged input tile)."""
    g = torch.Generator().manual_seed(7)
    K, N, R = 32, 128, 132
    A, Bfull = torch.randn((128, K), generator=g), torch.randn((R, K), generator=g)
    for j in range(5):
        strides = [128 * 16, 128, R * 16, 128, 2 * 128 * 16, 2 * R * 16, 0, j * 16]
        D = run_probe(img_kmajor(A), img_kmajor(Bfull), strides, K // 8, N)
        assert rel(D, A @ Bfull[j:j + N].t()) < 2e-3, (j, rel(D, A @ Bfull[j:j + N].t()))


@pytest.mark.xfail(reason="tf32 wgmma reads K-major operands only: the probe rejects MN-major ones (the weight gradient "
                          "kernels load their MN-major fragments with warp-level MMAs instead)", strict=False)
def test_mn_major_gemm():
    """Both operands MN-major (the weight-gradient form: reduction over time rows):
    D[m][n] = sum_k At[k][m] * Bt[k][n] with images [m/4][k][4]."""
    g = torch.Generator().manual_seed(9)
    Kt, N = 64, 128
    At, Bt = torch.randn((Kt, 128), generator=g), torch.randn((Kt, N), generator=g)
    a_img = At.reshape(Kt, 32, 4).permute(1, 0, 2).contiguous()        # [m/4][k][4]
    b_img = Bt.reshape(Kt, N // 4, 4).permute(1, 0, 2).contiguous()
    # MN-major, no swizzle: SBO = stride between 4-element MN groups (Kt*16 B), LBO = stride
    # between groups of 8 k-rows (128 B, contiguous); one K=8 step advances 8 rows = 128 B
    strides = [128, Kt * 16, 128, Kt * 16, 128, 128, 0, 0]
    D = run_probe(a_img, b_img, strides, Kt // 8, N, a_mn=1, b_mn=1)
    assert rel(D, At.t() @ Bt) < 2e-3, rel(D, At.t() @ Bt)


@pytest.mark.parametrize("shift", [1, 4, 20, 36, 132])
def test_tmem_load_at_any_start_column(shift):
    """The probe writes the accumulator from column `shift` on (any start column, not a multiple of 16): the
    persistent conv kernel stacks samples at a pitch of T+K-1 columns and reads every sample from its own first column."""
    from adaptive_voice_conversion_b200 import _lib as L
    N, K = 256, 16
    g = torch.Generator().manual_seed(shift)
    A, B = torch.randn((128, K), generator=g), torch.randn((N, K), generator=g)
    strides = [128 * 16, 128, N * 16, 128, 2 * 128 * 16, 2 * N * 16, 0, 0]
    lib = L.load()
    lib.avc_tc_probe_set_ld_shift(shift)
    try:
        D = run_probe(img_kmajor(A), img_kmajor(B), strides, K // 8, N)
    finally:
        lib.avc_tc_probe_set_ld_shift(0)
    ref = A @ B.t()
    hi = shift + ((N - shift) // 16) * 16                       # whole 16-column loads that fit in the allocation
    assert torch.isnan(D[:, :shift]).all()                      # untouched
    assert rel(D[:, shift:hi], ref[:, shift:hi]) < 2e-3, rel(D[:, shift:hi], ref[:, shift:hi])
