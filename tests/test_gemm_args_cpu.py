"""Argument validation of the GEMM entry points: a pointer or pitch the fused epilogue cannot use with its vector
accesses (float4 / uint2) is reported as DVT_ERR_INVALID with a message, before any CUDA call.

The pointers are fake integers: nothing is ever dereferenced.  The file runs only where there is no GPU, so that a
missing check shows up as DVT_ERR_CUDA (the call went on to the CUDA runtime, which finds no device) and fails cleanly,
instead of launching a kernel on misaligned memory."""
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: run on a machine without a GPU")

DVT_OK, DVT_ERR_INVALID, DVT_ERR_CUDA = 0, 1, 2
BF16, F32 = 0, 1

BASE = 1 << 32                      # 256-byte aligned fake device addresses, far apart
A, B, OUT, BIAS, GAMMA, PRE, BRANCH, LC = (BASE + i * (1 << 24) for i in range(8))


@pytest.fixture(scope="module")
def L():
    from dvt import _lib
    return _lib


@pytest.fixture(params=[0, 1], ids=["tensor_core", "simt"])
def impl(request, L):
    """Every check must hold on both implementations: the SIMT debug path shares the argument checks."""
    L.check(L.lib().dvt_set_debug_impl(request.param))
    yield request.param
    L.check(L.lib().dvt_set_debug_impl(-1))


def _expect_invalid(L, rc, *words):
    msg = L.lib().dvt_last_error().decode()
    assert rc == DVT_ERR_INVALID, f"expected DVT_ERR_INVALID, got {rc} ({msg})"
    for w in words:
        assert w in msg, f"message {msg!r} does not mention {w!r}"


def _gemm_tn(L, a=A, lda=64, b=B, ldb=64, dtype=BF16, M=128, N=128, K=64, bias=None, act=0, out=OUT, ldo=128,
             out_dtype=F32, splits=1):
    return L.lib().dvt_gemm_tn(a, lda, b, ldb, dtype, M, N, K, bias, act, out, ldo, out_dtype, splits, None)


def _residual(L, gamma=None, x=OUT, ldx=128, branch=None, ld_branch=128, bias=None):
    return L.lib().dvt_gemm_tn_residual(A, 64, B, 64, BF16, 128, 128, 64, bias, gamma, x, ldx, branch, ld_branch, None)


def _gemm_bf16(L, a=A, a_mn=0, b=B, b_mn=0, out=OUT, ldo=128, out_dtype=F32, splits=1, pre=None, ld_pre=0, lc=None,
               M=128, N=128, K=64):
    lda = ((M if a_mn else K) + 7) // 8 * 8       # 16-byte pitches
    ldb = ((N if b_mn else K) + 7) // 8 * 8
    return L.lib().dvt_gemm_bf16(a, lda, a_mn, b, ldb, b_mn, M, N, K, out, ldo, out_dtype, splits, pre, ld_pre, lc, None)


def _f32x3(L, a=A, b=B, out=OUT, lc=None, splits=1, N=128):
    return L.lib().dvt_gemm_f32x3(a, 64, 128 * 64, 0, b, 64, N * 64, 0, 128, N, 64, out, 128, splits, lc, None)


def test_valid_calls_reach_the_cuda_runtime(L, impl):
    """Controls: well-formed calls pass every check and fail only because there is no device."""
    for rc in (_gemm_tn(L), _gemm_tn(L, out_dtype=BF16, act=1, bias=BIAS), _gemm_tn(L, splits=3),
               _residual(L, gamma=GAMMA, branch=BRANCH, bias=BIAS),
               _gemm_bf16(L, pre=PRE, ld_pre=128, out_dtype=BF16), _gemm_bf16(L, a_mn=1, b_mn=1, lc=LC, N=129, ldo=128),
               _f32x3(L), _f32x3(L, lc=LC, N=129)):
        assert rc == DVT_ERR_CUDA, f"got {rc}: {L.lib().dvt_last_error().decode()}"


@pytest.mark.parametrize("off,out_dtype", [(4, F32), (8, F32), (12, F32), (2, BF16), (4, BF16)])
def test_misaligned_out(L, impl, off, out_dtype):
    _expect_invalid(L, _gemm_tn(L, out=OUT + off, out_dtype=out_dtype), "out", "aligned")


def test_bf16_out_needs_8_bytes_only(L, impl):
    assert _gemm_tn(L, out=OUT + 8, out_dtype=BF16) == DVT_ERR_CUDA


@pytest.mark.parametrize("off", [4, 8])
def test_misaligned_residual_out(L, impl, off):
    _expect_invalid(L, _residual(L, x=OUT + off), "out", "aligned")


@pytest.mark.parametrize("off", [4, 8, 12])
def test_misaligned_bias(L, impl, off):
    _expect_invalid(L, _gemm_tn(L, bias=BIAS + off, act=1, out_dtype=BF16), "bias", "aligned")
    _expect_invalid(L, _residual(L, bias=BIAS + off), "bias", "aligned")


@pytest.mark.parametrize("off", [4, 8])
def test_misaligned_gamma(L, impl, off):
    _expect_invalid(L, _residual(L, gamma=GAMMA + off), "gamma", "aligned")


@pytest.mark.parametrize("off", [2, 4])
def test_misaligned_branch(L, impl, off):
    _expect_invalid(L, _residual(L, branch=BRANCH + off), "branch", "aligned")


@pytest.mark.parametrize("off", [2, 4, 6])
def test_misaligned_gelu_preact(L, impl, off):
    _expect_invalid(L, _gemm_bf16(L, pre=PRE + off, ld_pre=128, out_dtype=BF16), "pre-activation", "aligned")


@pytest.mark.parametrize("ld_pre", [129, 130, 131])
def test_gelu_preact_pitch(L, impl, ld_pre):
    _expect_invalid(L, _gemm_bf16(L, pre=PRE, ld_pre=ld_pre, out_dtype=BF16), "pre-activation", "multiple of 4")


@pytest.mark.parametrize("off", [1, 2, 3])
def test_misaligned_last_col_out(L, impl, off):
    _expect_invalid(L, _gemm_bf16(L, a_mn=1, b_mn=1, lc=LC + off, N=129, ldo=128), "last_col_out", "aligned")
    _expect_invalid(L, _f32x3(L, lc=LC + off, N=129), "last_col_out", "aligned")


@pytest.mark.parametrize("which", ["A", "B"])
@pytest.mark.parametrize("off", [2, 8])
def test_misaligned_operands(L, impl, which, off):
    """Used to be checked only after the kernels' shared-memory set-up (and never on the SIMT path)."""
    kw = {"a": A + off} if which == "A" else {"b": B + off}
    _expect_invalid(L, _gemm_tn(L, **kw), "operands", "aligned")
    _expect_invalid(L, _gemm_bf16(L, **kw), "operands", "aligned")
    _expect_invalid(L, _f32x3(L, **kw), "operands", "aligned")


def test_operand_pitch(L, impl):
    _expect_invalid(L, _gemm_tn(L, lda=60), "pitch")
    _expect_invalid(L, _gemm_tn(L, ldb=66, dtype=F32), "pitch")
    _expect_invalid(L, L.lib().dvt_gemm_f32x3(A, 62, 128 * 64, 0, B, 64, 128 * 64, 0, 128, 128, 64, OUT, 128, 1, None,
                                              None), "pitches")


def test_layout_and_mode_checks(L, impl):
    _expect_invalid(L, _gemm_bf16(L, a_mn=1, b_mn=0), "not instantiated")
    _expect_invalid(L, _gemm_tn(L, ldo=130), "ldo")
    _expect_invalid(L, _gemm_bf16(L, a_mn=1, b_mn=1, lc=LC, N=128), "last_col_out")   # (N - 1) % 4 != 0
    _expect_invalid(L, _gemm_tn(L, M=0), "empty shape")


def test_split_k_rejects_bias(L, impl):
    """Every split runs the epilogue on its own partial sum: a bias would be added `splits` times."""
    _expect_invalid(L, _gemm_tn(L, splits=2, bias=BIAS), "split-K", "bias")
