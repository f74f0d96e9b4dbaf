"""The persistent wgmma GEMM (gemm_persistent.cu) at chosen, uneven per-expert row counts in the scatter layout, with every unused row
of an expert's input segment poisoned with NaN.  The kernel loads token rows in 16-row boxes, only as many as an expert has, and stores
only valid token columns from the register epilogue: a wrong transaction count, a box-count off-by-one or a stored garbage column shows
up here as a hang, a NaN or a written padding row."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -4096.0   # exact in bf16 and fp32
# every box (16 rows) and epilogue chunk (64 rows) boundary, from both sides; the second set also spans two 64-row token tiles
COUNTS = {64: [0, 1, 6, 15, 16, 17, 31, 33, 63, 64], 128: [0, 1, 6, 15, 16, 17, 31, 33, 63, 64, 65, 97, 127, 128]}


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(torch.bfloat16)


def scatter_input(counts, stride, K, seed):
    x = rnd(len(counts) * stride, K, seed=seed)
    for e, c in enumerate(counts):
        x[e * stride + c:(e + 1) * stride] = float("nan")
    return x


def reference(x, w, w2, counts, stride):
    """fp32 result of each valid row, keyed by its row in the scatter layout."""
    out = {}
    for e, c in enumerate(counts):
        if c == 0:
            continue
        xs = x[e * stride:e * stride + c].float()
        y = xs @ w[e].float().t()
        if w2 is not None:
            y = torch.nn.functional.silu(y) * (xs @ w2[e].float().t())
        out[e] = y
    return out


def check_rows(got, ref, counts, stride):
    for e, y in ref.items():
        g = got[e * stride:e * stride + counts[e]].float()
        assert torch.isfinite(g).all(), f"expert {e}: non-finite output"
        err = (g - y).abs().max().item()
        assert err < 2e-2 * max(1.0, y.abs().max().item()), (e, counts[e], err)


@pytest.mark.parametrize("stride", [64, 128])
@pytest.mark.parametrize("K,N,dual", [(2048, 1408, True), (1408, 2048, False)])
def test_grouped_scatter_uneven_counts(stride, K, N, dual):
    from mlx_sharding_b200.ops import b200

    C = b200.load_extension()
    counts_l = COUNTS[stride]
    E = len(counts_l)
    counts = torch.tensor(counts_l, dtype=torch.int32, device=DEV)
    x = scatter_input(counts_l, stride, K, seed=1)
    w = rnd(E, N, K, scale=0.03, seed=2)
    w2 = rnd(E, N, K, scale=0.03, seed=3) if dual else None
    ref = reference(x, w, w2, counts_l, stride)
    total = int(counts.sum())
    out_fp32 = not dual
    odt = torch.float32 if out_fp32 else torch.bfloat16

    got = C.grouped_linear(x, w, w2, counts, stride, 1 if dual else 0, out_fp32, None, None, None, total, stride)
    assert got.dtype == odt and got.shape == (E * stride, N)
    check_rows(got, ref, counts_l, stride)

    # Row-address return path: every row of the layout (padding rows included) points into a sentinel-filled buffer, so a row
    # outside the counts that gets written is visible.  The completion flag is a local counter bumped once per launch.
    dst = torch.full((E * stride, N), SENTINEL, dtype=odt, device=DEV)
    row_dst = dst.data_ptr() + torch.arange(E * stride, dtype=torch.int64, device=DEV) * (N * dst.element_size())
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    peers = torch.tensor([flag.data_ptr()], dtype=torch.int64, device=DEV)
    done = torch.zeros(1, dtype=torch.int32, device=DEV)
    empty = C.grouped_linear(x, w, w2, counts, stride, 1 if dual else 0, out_fp32, row_dst, peers, done, total, stride)
    torch.cuda.synchronize()
    assert empty.numel() == 0
    assert int(flag.item()) == 1 and int(done.item()) == 0
    check_rows(dst, ref, counts_l, stride)
    valid = torch.zeros(E * stride, dtype=torch.bool, device=DEV)
    for e, c in enumerate(counts_l):
        valid[e * stride:e * stride + c] = True
    assert (dst[~valid].float() == SENTINEL).all(), "a row outside the per-expert counts was written"
    # both routes store the same values
    assert torch.equal(dst[valid], got[valid])


@pytest.mark.parametrize("T", [5, 37, 100, 300])
def test_dense_persistent_partial_tiles(T):
    """Un-grouped persistent launches (token tiles of 16, 64 and 128 rows, last tile partial) with bias, SiLU-gating and residual."""
    from mlx_sharding_b200.ops import b200

    C = b200.load_extension()
    K, N = 2048, 1408
    x = rnd(T, K, seed=1)
    w, w2 = rnd(N, K, scale=0.03, seed=2), rnd(N, K, scale=0.03, seed=3)
    bias, res = rnd(N, scale=0.5, seed=4), rnd(T, N, seed=5)
    got = C.linear(x, w, w2, None, bias, 1, 0.0, False, None, 1)
    g = x.float() @ w.float().t() + bias.float()
    ref = torch.nn.functional.silu(g) * (x.float() @ w2.float().t())
    assert torch.isfinite(got.float()).all()
    assert (got.float() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())
    got = C.linear(x, w, None, res, None, 0, 0.0, True, None, 1)
    ref = x.float() @ w.float().t() + res.float()
    assert (got - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())
