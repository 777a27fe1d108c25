"""GPU checks of the GEMM engine's TMA-loaded residual (bf16 staged epilogue).

A bf16-output call whose residual TMA can address has the residual tile loaded into the staging buffer under the MMAs
and added from shared memory.  Every case here is compared bit for bit with the register epilogue
(E4T_GEMM_EPI_PLAIN=0), which reads the residual from global memory, and with an fp32 restatement at the bf16-output
tolerance of test_gemm_gpu.py (inputs are bf16-representable; the difference is accumulation order and the final
rounding).  The shapes cover the UNet / ViT residual calls, M and N tails, every tile width, batched, strided and
misaligned residuals (the last takes the global-memory read), the implicit convolutions, and launches with one and
with many tiles per CTA.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
torch.backends.cuda.matmul.allow_tf32 = False


def _rel(a, b):
    a = a.float(); b = b.float()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-12)).item()


def _mk(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _staged_and_plain(monkeypatch, fn):
    """fn() with the staged epilogue, then with the register epilogue; both outputs."""
    monkeypatch.delenv("E4T_GEMM_EPI_PLAIN", raising=False)
    staged = fn()
    monkeypatch.setenv("E4T_GEMM_EPI_PLAIN", "0")
    plain = fn()
    monkeypatch.delenv("E4T_GEMM_EPI_PLAIN")
    torch.cuda.synchronize()
    return staged, plain


def _check_gemm(monkeypatch, M, N, K, *, seed, bias=True, rowgroup=False, alpha=1.0, force_bn=0, res_view=None):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = _mk((M, K), g, K ** -0.5); B = _mk((N, K), g)
    bs = torch.randn(N, generator=g, device="cuda") if bias else None
    rpg = 100
    rg = torch.randn((M + rpg - 1) // rpg, N, generator=g, device="cuda") if rowgroup else None
    res = res_view(g) if res_view is not None else _mk((M, N), g)
    staged, plain = _staged_and_plain(monkeypatch, lambda: ops.gemm(
        A, B, bias=bs, rowgroup=rg, rows_per_group=rpg, residual=res, alpha=alpha, force_bn=force_bn))
    ref = alpha * (A.float() @ B.float().t()) + res.float()
    if bias:
        ref = ref + bs
    if rowgroup:
        ref = ref + rg.repeat_interleave(rpg, 0)[:M]
    assert torch.equal(staged, plain)
    assert _rel(staged, ref) < 4e-3, _rel(staged, ref)


# UNet residual calls at B = 2 (to_out / FF2 / proj_out of levels 0-3), a ViT-H-like M, an M tail that ends inside
# the second MMA warpgroup's rows and one that leaves it no rows, an N tail that is not a whole 32-column box
@pytest.mark.parametrize("M,N,K", [(8192, 320, 320), (8192, 320, 1280), (2048, 640, 640), (2048, 640, 2560),
                                   (512, 1280, 1280), (128, 1280, 1280), (4112, 1280, 5120), (1000, 320, 320),
                                   (960, 640, 320), (1000, 328, 320)])
def test_gemm_residual_shapes(monkeypatch, M, N, K):
    _check_gemm(monkeypatch, M, N, K, seed=M + 3 * N + 7 * K)


@pytest.mark.parametrize("bn", [64, 96, 128, 160, 192, 224, 256])
def test_gemm_residual_tile_widths(monkeypatch, bn):
    _check_gemm(monkeypatch, 1000, 328, 192, seed=bn, rowgroup=True, alpha=0.5, force_bn=bn)


def test_gemm_residual_batched(monkeypatch):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(11)
    bt, M, N, K = 3, 520, 320, 256
    A = _mk((bt, M, K), g, K ** -0.5); B = _mk((N, K), g)
    res = _mk((bt, M, N), g)
    bs = torch.randn(N, generator=g, device="cuda")
    staged, plain = _staged_and_plain(monkeypatch, lambda: ops.gemm(A, B, bias=bs, residual=res))
    ref = A.float() @ B.float().t() + bs + res.float()
    assert torch.equal(staged, plain)
    assert _rel(staged, ref) < 4e-3


def test_gemm_residual_column_slice(monkeypatch):
    """A residual that is a column slice of a wider buffer: row pitch ldr > N."""
    M, N = 1000, 320

    def view(g):
        return _mk((M, 2 * N + 64), g)[:, 64:64 + N]
    _check_gemm(monkeypatch, M, N, 320, seed=12, res_view=view)


def test_gemm_residual_misaligned(monkeypatch):
    """A residual whose base is 8 bytes off a 16-byte boundary: TMA cannot address it, the epilogue reads it."""
    M, N = 1000, 320

    def view(g):
        r = _mk((M * N + 8,), g)[4:4 + M * N].view(M, N)
        assert r.data_ptr() % 16 == 8
        return r
    _check_gemm(monkeypatch, M, N, 320, seed=13, res_view=view)


def test_gemm_residual_tiles_per_cta(monkeypatch):
    """65536 x 320 (level 0 at B = 16): several tiles per CTA, so the residual barriers' phases wrap; 128 x 128: a
    single tile."""
    _check_gemm(monkeypatch, 65536, 320, 320, seed=14)
    _check_gemm(monkeypatch, 128, 128, 64, seed=15)


@pytest.mark.parametrize("entry,H,W", [("conv3x3", 32, 32), ("conv3x3_im2col", 32, 32), ("conv3x3_im2col", 24, 40)])
def test_conv3x3_residual(monkeypatch, entry, H, W):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(H * W)
    Bn, Cin, Cout = 2, 320, 320
    x = _mk((Bn, H, W, Cin), g)
    w9 = _mk((9, Cout, Cin), g, (9 * Cin) ** -0.5)
    bias = torch.randn(Cout, generator=g, device="cuda")
    temb = torch.randn(Bn, Cout, generator=g, device="cuda")
    res = _mk((Bn, H, W, Cout), g)
    fn = getattr(ops, entry)
    staged, plain = _staged_and_plain(monkeypatch, lambda: fn(x, w9, bias=bias, rowgroup=temb, residual=res))
    w = w9.float().view(3, 3, Cout, Cin).permute(2, 3, 0, 1)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w, bias, padding=1).permute(0, 2, 3, 1)
    ref = ref + temb[:, None, None, :] + res.float()
    assert torch.equal(staged, plain)
    assert _rel(staged, ref) < 4e-3, _rel(staged, ref)
