"""GPU tests of the normalisation and gated-activation kernels (GroupNorm-NHWC, LayerNorm, RMSNorm, SwiGLU / GEGLU)
against float64 statements of the same operations on the same rounded inputs, at the inputs where such kernels go
wrong: rows and groups whose mean is large next to their spread, rows with a few huge ("massive") columns, near-constant
and constant groups, and every dispatch branch (warp / block / register kernels, ragged tails, column-sliced grids).

Notation: u_T is the unit roundoff of the element type T (2^-24 fp32, 2^-11 fp16, 2^-8 bf16); u = 2^-24 is fp32's.
For a row or group, mu and sigma are its mean and (biased) standard deviation, r = 1 / sqrt(sigma^2 + eps), xhat =
(x - mu) r, and A = max |x| over the row or group -- the largest magnitude the kernel's fp32 sums see.

GroupNorm and LayerNorm (y = gamma xhat + beta, rounded once to T):
  * the kernels form mu and r in fp32.  A stable method (centred or shifted sums, pairwise merges) gets mu to within a
    few u A -- rounding the mean itself to fp32 costs u |mu| -- and r to within a few u relative.  An error d in mu moves
    xhat by d r, so the statistics contribute c u (A r + |xhat|) |gamma|, plus u |beta| for the fp32 fma, with c = 16
    (several times the worst fixed-order sum seen here).  The term is linear in the conditioning A r ~ 1 + |mu| / sigma;
    the one-pass variance E[x^2] - mu^2 instead loses (mu / sigma)^2 ulps and fails it from mu / sigma ~ 16 on in fp32;
  * the final rounding adds u_T |ref|, and u_T times the smallest normal number below it.
  With SiLU (GroupNorm): the normalised value is rounded to T first, so its error (the bound above) is carried through
  silu with a factor |silu'(ref)| + 0.05 (silu'' <= 0.5 over an interval of width < 0.1), the fast-math silu
  (__expf, __fdividef) errs by < 2^-19 relative at the |n| < 16 seen here, and the result is rounded to T.
  GroupNorm applies y = x (r gamma) + (beta - mu r gamma): the folded shift's rounding, u |mu| r |gamma|, is inside
  the statistics term.

RMSNorm (y = round_T(w round_T(x r))): r is the only fp32 statistic, within 2^-18 relative of the float64 one (rsqrtf's
  2 ulp plus a sum of squares of <= 64 terms per thread and a 10-level tree).  Rounding is monotone, so the kernel's
  intermediate is round_T(x r (1 +- 2^-18)) -- one of two adjacent values -- and, since w * v of two 16-bit values is
  exact in fp32, the 16-bit output is round_T(w v) for one of them: every element is bit-exact against one of two
  candidates, and >= 99 % against the reference's own rounding points.  fp32: |err| <= (2^-18 + 2 u) |ref|.

SwiGLU / GEGLU (out = round_T(round_T(act(g)) up)): the activation is computed in fp32 and is within e of the float64 one:
  silu, 16-bit (__expf, __fdividef): e = (2^-20 + |g| 2^-23) |act| -- __expf rounds g log2(e) to fp32, a relative error
  of ~|g| 2^-24 in the result; silu, fp32 (expf, IEEE division): e = 2^-21 |act|; gelu (erff, both): e = 2^-21 (|g| +
  |act|) -- erff's 2 ulp is an absolute error next to 1, which 1 + erf exposes in the negative tail.  Below 2^-100,
  where 1 + exp(-g) overflows and the division returns 0, e is absolute.  Rounding is monotone and the 16-bit product
  is exact in fp32, so every output lies between round_T(lo * up) and round_T(hi * up) with lo, hi = round_T(act -+ e);
  fp32 adds the product's rounding u.

Backward (LayerNorm, RMSNorm): the bounds of tests/test_train_kernels_gpu.py, plus for LayerNorm the same statistics
term as the forward carried through dx = r (g - mean(g) - xhat mean(g xhat)) and dweight = sum dy xhat."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DTYPES = [F32, F16, BF16]
U = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}
U32 = 2.0 ** -24
SUB = {t: U[t] * torch.finfo(t).smallest_normal for t in U}
C_STAT = 16
TINY = 2.0 ** -100


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ops():
    from mm_interleaved_b200 import ops
    return ops


def _near_constant(mu0, n, dtype, g):
    """Values mu0 + k ulp(mu0), k in -2..2: a spread of ~1.4 ulp, far below sqrt(eps) for the mu0 used here."""
    if dtype == F32:
        return mu0 + 1e-4 * torch.randn(n, generator=g, dtype=torch.float64)
    ulp = mu0 * 2.0 * U[dtype]
    return mu0 + ulp * torch.randint(-2, 3, (n,), generator=g).double()


NEAR_CONST_MU = {F32: 8.0, F16: 2.0 ** -2, BF16: 2.0 ** -6}


def _affine_bound(dtype, ref, xhat, ar, w, b):
    """u_T |ref| + c u (A r + |xhat|) |gamma| + c u |beta| (+ the subnormal floor), elementwise."""
    gam = w.abs() if w is not None else 1.0
    bet = b.abs() if b is not None else 0.0
    stat = C_STAT * U32 * (gam * (ar + xhat.abs()) + bet)
    return U[dtype] * ref.abs() + (1 + U[dtype]) * stat + SUB[dtype]


def _silu64(n):
    return n * torch.sigmoid(n)


def _dsilu64(n):
    s = torch.sigmoid(n)
    return s * (1 + n * (1 - s))


def _report(err, bound):
    i = int((err - bound).argmax())
    return f"max err {err.max().item():.3e}; worst excess at {i}: err {err.flatten()[i].item():.3e} > {bound.flatten()[i].item():.3e}"


# ---------------------------------------------------------------------------------------------------------- GroupNorm
def _gn_check(x, G, w, b, eps, silu, out):
    """x, w, b: CPU tensors of the element type (the kernel's inputs); out: the kernel's output."""
    dtype = x.dtype
    B, C = x.shape[:2]
    xd = x.double()
    wd = w.double() if w is not None else None
    bd = b.double() if b is not None else None
    ref = F.group_norm(xd, G, wd, bd, eps)
    grp = xd.reshape(B, G, -1)
    mu, var, amax = grp.mean(-1), grp.var(-1, unbiased=False), grp.abs().amax(-1)
    r = torch.rsqrt(var + eps)
    per_c = lambda t: t.repeat_interleave(C // G, dim=1)[:, :, None, None]
    xhat = (xd - per_c(mu)) * per_c(r)
    shape_c = (1, C, 1, 1)
    bound = _affine_bound(dtype, ref, xhat, per_c(amax * r), wd.view(shape_c) if wd is not None else None,
                          bd.view(shape_c) if bd is not None else None)
    del xhat
    if silu:
        ref_s = _silu64(ref)
        bound = ((U[dtype] + 2.0 ** -19) * ref_s.abs() + (1 + U[dtype]) * (_dsilu64(ref).abs() + 0.05) * bound
                 + SUB[dtype] + TINY)
        ref = ref_s
    got = out.cpu().double()
    err = (got - ref).abs()
    assert bool((err <= bound).all()), _report(err, bound)


def _gn_run(x, G, w, b, eps, silu):
    ops = _ops()
    xd = x.to(DEV).contiguous(memory_format=torch.channels_last)
    wd = w.to(DEV) if w is not None else None
    bd = b.to(DEV) if b is not None else None
    out = ops.group_norm_nhwc(xd, G, wd, bd, eps, silu=silu)
    again = ops.group_norm_nhwc(xd, G, wd, bd, eps, silu=silu)
    torch.cuda.synchronize()
    assert out.dtype == x.dtype and out.shape == x.shape and out.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(out, again), "two runs of group_norm_nhwc differ"
    return out


def _gn_affine(C, dtype, g):
    w = (1 + 0.2 * torch.randn(C, generator=g)).to(dtype)
    b = (0.2 * torch.randn(C, generator=g)).to(dtype)
    return w, b


def _gn_offsets(B, G, C, max_ratio, sigma, g):
    """Per-group means of either sign, |mu| / sigma spread over [0, max_ratio], as a (B, C, 1, 1) tensor."""
    sign = torch.randint(0, 2, (B, G), generator=g).double() * 2 - 1
    mag = torch.rand(B, G, generator=g, dtype=torch.float64) * max_ratio * sigma
    return (sign * mag).repeat_interleave(C // G, dim=1)[:, :, None, None]


# (mean / sigma, sigma) of every group: fp32 reaches 4096; the 16-bit types stop where a group's values would collapse
# onto a few representable numbers (bf16 64 +- 0.5 z, fp16 256 +- z)
GN_CONDITIONING = [(F32, 0, 1.0), (F32, 16, 1.0), (F32, 256, 1.0), (F32, 4096, 1.0),
                   (F16, 0, 1.0), (F16, 16, 1.0), (F16, 256, 1.0),
                   (BF16, 0, 1.0), (BF16, 16, 0.5), (BF16, 128, 0.5)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("dtype,ratio,sigma", GN_CONDITIONING)
def test_group_norm_at_offset_groups(dtype, ratio, sigma, silu):
    B, C, H, W, G = 2, 320, 32, 32, 32
    g = _gen(ratio * 7 + int(silu) + 100 * DTYPES.index(dtype))
    sign = (torch.randint(0, 2, (B, G), generator=g).double() * 2 - 1).repeat_interleave(C // G, dim=1)[:, :, None, None]
    x = (sign * ratio * sigma + sigma * torch.randn(B, C, H, W, generator=g, dtype=torch.float64)).to(dtype)
    w, b = _gn_affine(C, dtype, g)
    _gn_check(x, G, w, b, 1e-5, silu, _gn_run(x, G, w, b, 1e-5, silu))


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("dtype", DTYPES)
def test_group_norm_near_constant_and_constant_groups(dtype, eps):
    """Groups 0..7: near-constant (sigma^2 << eps); 8..15: exactly constant (the reference is beta); the rest ordinary."""
    B, C, H, W, G = 2, 320, 16, 16, 32
    cg = C // G
    g = _gen(int(1e6 * eps) + DTYPES.index(dtype))
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    consts = torch.tensor([3.0, -0.75, 17.0, 0.125, -40.0, 1.0, 6.5, -2.25], dtype=torch.float64)
    for bi in range(B):
        for gi in range(8):
            n = cg * H * W
            mu0 = NEAR_CONST_MU[dtype] * (1 if gi % 2 == 0 else -1)
            x[bi, gi * cg:(gi + 1) * cg] = _near_constant(mu0, n, dtype, g).view(cg, H, W)
            x[bi, (8 + gi) * cg:(9 + gi) * cg] = consts[gi]
    x = x.to(dtype)
    w, b = _gn_affine(C, dtype, g)
    out = _gn_run(x, G, w, b, eps, False)
    _gn_check(x, G, w, b, eps, False, out)


GN_SHAPES = [
    ((2, 320, 32, 32), 32, True), ((3, 64, 16, 16), 32, False), ((2, 960, 8, 8), 32, True),
    ((1, 2560, 8, 8), 32, True), ((2, 1920, 16, 16), 32, False),
    ((2, 320, 33, 17), 32, True),          # ragged H*W: chunk and unroll tails
    ((3, 64, 7, 9), 32, False),            # fewer pixels than a chunk's lanes * 4
    ((2, 96, 16, 16), 32, True),           # a group of 3 channels, narrower than one 16-byte vector
]
GN_BIG_SHAPES = [
    ((16, 320, 64, 64), 32, True),         # the denoise step's batch with classifier-free guidance
    ((1, 128, 512, 512), 32, False),       # the VAE decoder's top level: 64 chunks of 4096 pixels
]


def _gn_shape_case(shape, G, silu, dtype, seed):
    B, C, H, W = shape
    g = _gen(seed)
    off = _gn_offsets(B, G, C, 16.0, 1.0, g)
    x = (off + torch.randn(shape, generator=g, dtype=torch.float64)).to(dtype)
    w, b = _gn_affine(C, dtype, g)
    _gn_check(x, G, w, b, 1e-5, silu, _gn_run(x, G, w, b, 1e-5, silu))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape,G,silu", GN_SHAPES)
def test_group_norm_shapes(shape, G, silu, dtype):
    """Groups with means spread over [-16, 16] sigma at every shape the UNet and VAE use, and the ragged ones."""
    _gn_shape_case(shape, G, silu, dtype, sum(shape) + DTYPES.index(dtype))


@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("shape,G,silu", GN_BIG_SHAPES)
def test_group_norm_large_maps(shape, G, silu, dtype):
    _gn_shape_case(shape, G, silu, dtype, sum(shape) + DTYPES.index(dtype))


@pytest.mark.parametrize("affine", ["none", "weight", "bias"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_group_norm_without_weight_or_bias(dtype, affine):
    B, C, H, W, G = 2, 320, 16, 16, 32
    g = _gen(DTYPES.index(dtype) + 17)
    x = (_gn_offsets(B, G, C, 16.0, 1.0, g) + torch.randn(B, C, H, W, generator=g, dtype=torch.float64)).to(dtype)
    w, b = _gn_affine(C, dtype, g)
    w = w if affine == "weight" else None
    b = b if affine == "bias" else None
    _gn_check(x, G, w, b, 1e-5, True, _gn_run(x, G, w, b, 1e-5, True))


# ---------------------------------------------------------------------------------------------------------- LayerNorm
def _ln_rows(rows, cols, dtype, g):
    """Row kinds, cycling: ordinary (0.5 + z), offset +-30 sigma, offset +-1000 sigma, four massive columns at +-1000
    sigma (CLIP's outlier channels), near-constant, exactly constant."""
    x = torch.empty(rows, cols, dtype=torch.float64)
    for i in range(rows):
        kind = i % 6
        z = torch.randn(cols, generator=g, dtype=torch.float64)
        sign = 1.0 if (i // 6) % 2 == 0 else -1.0
        if kind == 0:
            x[i] = 0.5 + z
        elif kind == 1:
            x[i] = sign * 30 + z
        elif kind == 2:
            x[i] = sign * 1000 + z
        elif kind == 3:
            idx = torch.randperm(cols, generator=g)[:4]
            z[idx] = torch.tensor([1e3, -1e3, 1e3, -1e3], dtype=torch.float64)
            x[i] = z
        elif kind == 4:
            x[i] = _near_constant(sign * NEAR_CONST_MU[dtype], cols, dtype, g)
        else:
            x[i] = sign * 2.5
    return x.to(dtype)


def _ln_check(x, w, b, eps, out):
    dtype = x.dtype
    xd = x.double()
    wd = w.double() if w is not None else None
    bd = b.double() if b is not None else None
    ref = F.layer_norm(xd, (xd.shape[-1],), wd, bd, eps)
    mu, var = xd.mean(-1, keepdim=True), xd.var(-1, unbiased=False, keepdim=True)
    r = torch.rsqrt(var + eps)
    bound = _affine_bound(dtype, ref, (xd - mu) * r, xd.abs().amax(-1, keepdim=True) * r, wd, bd)
    err = (out.cpu().double() - ref).abs()
    assert bool((err <= bound).all()), _report(err, bound)


def _ln_case(rows, cols, dtype, eps, with_w=True, with_b=True, seed=0, misaligned=False):
    ops = _ops()
    g = _gen(seed)
    x = _ln_rows(rows, cols, dtype, g)
    w = (1 + 0.2 * torch.randn(cols, generator=g)).to(dtype) if with_w else None
    b = (0.2 * torch.randn(cols, generator=g)).to(dtype) if with_b else None
    if misaligned:            # contiguous, but one element past a 16-byte boundary: the block kernel's path
        buf = torch.empty(rows * cols + 1, dtype=dtype, device=DEV)
        xd = buf[1:].view(rows, cols)
        xd.copy_(x.to(DEV))
        assert xd.is_contiguous() and xd.data_ptr() % 16 != 0
    else:
        xd = x.to(DEV)
    wd = w.to(DEV) if w is not None else None
    bd = b.to(DEV) if b is not None else None
    out = ops.layernorm(xd, wd, bd, eps)
    again = ops.layernorm(xd, wd, bd, eps)
    torch.cuda.synchronize()
    assert torch.equal(out, again)
    _ln_check(x, w, b, eps, out)


# 16-bit: cols 64 / 320 / 1024 / 2048 take the warp kernel with 1 / 2 / 4 / 8 vectors per lane; fp32: 64 / 256 / 320 /
# 1024 take 1 / 2 / 4 / 8 and 2048 the block kernel.  100 (16-bit: not a multiple of the vector) and 5120 (too long)
# take the block kernel.
LN_COLS = [64, 100, 256, 320, 1024, 2048, 5120]


@pytest.mark.parametrize("cols", LN_COLS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_layernorm_forward(dtype, cols):
    _ln_case(6 * 8 + 3, cols, dtype, 1e-5, seed=cols + DTYPES.index(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
def test_layernorm_forward_eps_1e6_and_misaligned_rows(dtype):
    _ln_case(6 * 4 + 1, 768, dtype, 1e-6, seed=5 + DTYPES.index(dtype))
    _ln_case(6 * 4 + 1, 768, dtype, 1e-6, seed=6 + DTYPES.index(dtype), misaligned=True)


@pytest.mark.parametrize("with_w,with_b", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("cols", [320, 100])
@pytest.mark.parametrize("dtype", DTYPES)
def test_layernorm_forward_without_weight_or_bias(dtype, cols, with_w, with_b):
    _ln_case(6 * 2, cols, dtype, 1e-5, with_w, with_b, seed=cols + 3)


# ------------------------------------------------------------------------------------------------------------ RMSNorm
def _rms_rows(rows, cols, g):
    """Ordinary rows, rows scaled by 1e-3 and 1e3, rows with four massive columns, and all-zero rows."""
    x = torch.randn(rows, cols, generator=g, dtype=torch.float64)
    for i in range(rows):
        kind = i % 5
        if kind == 1:
            x[i] *= 1e-3
        elif kind == 2:
            x[i] *= 1e3
        elif kind == 3:
            x[i, torch.randperm(cols, generator=g)[:4]] = torch.tensor([1e3, -1e3, 1e3, -1e3], dtype=torch.float64)
        elif kind == 4:
            x[i] = 0.0
    return x


# fp32: 1024 / 4096 take the single-pass register kernel, 5120 the block kernel; 16-bit: 4096 / 5120 / 8192 the
# register kernel, 10240 the block kernel
RMS_CASES = [(F32, 1024), (F32, 4096), (F32, 5120), (F16, 4096), (F16, 8192), (F16, 10240),
             (BF16, 4096), (BF16, 5120), (BF16, 8192), (BF16, 10240)]
RMS_EPS_REL = 2.0 ** -18


@pytest.mark.parametrize("dtype,cols", RMS_CASES)
def test_rmsnorm_forward_matches_rounding_points(dtype, cols):
    ops = _ops()
    rows, eps = 5 * 7 + 2, 1e-6
    g = _gen(cols + DTYPES.index(dtype))
    x = _rms_rows(rows, cols, g).to(dtype)
    w = (1 + 0.2 * torch.randn(cols, generator=g)).to(dtype)
    out = ops.rmsnorm(x.to(DEV), w.to(DEV), eps)
    torch.cuda.synchronize()
    y = out.cpu()
    assert torch.isfinite(y).all()
    zero_rows = (x == 0).all(-1)
    assert zero_rows.any() and bool((y[zero_rows] == 0).all()), "an all-zero row must give exactly 0"

    xd, wd = x.double(), w.double()
    a = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    if dtype == F32:
        ref = wd * a
        err = (y.double() - ref).abs()
        bound = (RMS_EPS_REL + 2 * U32) * ref.abs() + SUB[F32]
        assert bool((err <= bound).all()), _report(err, bound)
        return
    exact = (wd * a.to(dtype).double()).to(dtype)                     # the reference's rounding points
    lo = (wd * (a * (1 - RMS_EPS_REL)).to(dtype).double()).to(dtype)
    hi = (wd * (a * (1 + RMS_EPS_REL)).to(dtype).double()).to(dtype)
    ok = (y == lo) | (y == hi)
    assert bool(ok.all()), f"{int((~ok).sum())} elements off both candidates, e.g. got {y[~ok][:4]} want {lo[~ok][:4]} / {hi[~ok][:4]}"
    assert (y == exact).double().mean().item() >= 0.99


# ----------------------------------------------------------------------------------------------------- SwiGLU / GEGLU
def _glu_err(act_name, dtype, gate, act):
    if act_name == "gelu":
        return 2.0 ** -21 * (gate.abs() + act.abs()) + TINY
    if dtype == F32:
        return 2.0 ** -21 * act.abs() + TINY
    return (2.0 ** -20 + gate.abs() * 2.0 ** -23) * act.abs() + TINY


@pytest.mark.parametrize("act_name", ["silu", "gelu"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,inter", [(1, 13824), (2, 13824), (7, 13824), (1, 5120), (2, 5120), (7, 5120),
                                        (160, 5120)])
def test_glu_at_decode_shapes(rows, inter, dtype, act_name):
    """Few rows (a decode step: the row is cut into column slices, gridDim.y > 1) and rows >= the SM count (one slice);
    gates spanning +-90 (saturation, overflow of exp(-g), the fast division's range)."""
    ops = _ops()
    g = _gen(rows * 31 + inter + DTYPES.index(dtype))
    gate = torch.where(torch.rand(rows, inter, generator=g) < 0.5,
                       180 * torch.rand(rows, inter, generator=g, dtype=torch.float64) - 90,
                       3 * torch.randn(rows, inter, generator=g, dtype=torch.float64)).to(dtype)
    up = torch.randn(rows, inter, generator=g).to(dtype)
    if act_name == "silu":
        packed = torch.cat([gate, up], -1)                            # [gate | up]
        out = ops.swiglu(packed.to(DEV))
    else:
        packed = torch.cat([up, gate], -1)                            # [value | gate]
        out = ops.geglu(packed.to(DEV))
    torch.cuda.synchronize()
    y = out.cpu().double()
    gd, ud = gate.double(), up.double()
    act = _silu64(gd) if act_name == "silu" else 0.5 * gd * (1 + torch.special.erf(gd * 0.5 ** 0.5))
    e = _glu_err(act_name, dtype, gd, act)
    if dtype == F32:
        a_lo, a_hi = act - e, act + e
    else:
        a_lo, a_hi = (act - e).to(dtype).double(), (act + e).to(dtype).double()
    p1, p2 = a_lo * ud, a_hi * ud
    lo, hi = torch.minimum(p1, p2), torch.maximum(p1, p2)
    if dtype == F32:
        lo, hi = lo - U32 * lo.abs() - SUB[F32], hi + U32 * hi.abs() + SUB[F32]
    else:
        lo, hi = lo.to(dtype).double(), hi.to(dtype).double()
    ok = (y >= lo) & (y <= hi)
    assert bool(ok.all()), f"{int((~ok).sum())} outputs outside their interval, e.g. g={gd[~ok][:3]} got {y[~ok][:3]} in [{lo[~ok][:3]}, {hi[~ok][:3]}]"
    if dtype != F32:
        # bit identity with round_T(round_T(act(g)) * up) wherever the fp32 activation is accurate next to T's rounding
        # (not gelu's negative tail, where 1 + erff(g / sqrt 2) cancels: erff is -1 exactly below g ~ -5.9)
        exact = (act.to(dtype).double() * ud).to(dtype).double()
        sharp = e <= 2.0 ** -4 * U[dtype] * act.abs()
        assert sharp.double().mean().item() >= 0.5                    # ~0.6 (gelu) / ~0.9 (silu) of these gates
        assert (y == exact)[sharp].double().mean().item() >= 0.99


# ----------------------------------------------------------------------------------------------------------- backward
def _offset_massive_rows(rows, cols, g):
    """Ordinary, offset +-30 and +-300 sigma, and four massive columns at +-300 sigma, cycling."""
    x = torch.randn(rows, cols, generator=g, dtype=torch.float64)
    for i in range(rows):
        kind, sign = i % 4, (1.0 if (i // 4) % 2 == 0 else -1.0)
        if kind == 1:
            x[i] += sign * 30
        elif kind == 2:
            x[i] += sign * 300
        elif kind == 3:
            x[i, torch.randperm(cols, generator=g)[:4]] = torch.tensor([300.0, -300.0, 300.0, -300.0], dtype=torch.float64)
    return x


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("cols", [64, 768])
def test_layernorm_backward_at_offset_and_massive_rows(cols, dtype):
    ops = _ops()
    rows, eps, u = 4 * 40 + 3, 1e-6, U[dtype]
    g = _gen(cols + DTYPES.index(dtype))
    x = _offset_massive_rows(rows, cols, g).to(dtype)
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(dtype)
    dy = torch.randn(rows, cols, generator=g).to(dtype)
    with torch.no_grad():
        dx, dw, db = ops.layernorm_backward(x.to(DEV), w.to(DEV), dy.to(DEV), eps)
    torch.cuda.synchronize()

    x64, w64, b64 = x.double().requires_grad_(True), w.double().requires_grad_(True), torch.zeros(cols, dtype=torch.float64, requires_grad=True)
    F.layer_norm(x64, (cols,), w64, b64, eps).backward(dy.double())
    xd, wd, dyd = x.double(), w.double(), dy.double()
    r = torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
    xh = (xd - xd.mean(-1, keepdim=True)) * r
    gg = (dyd * wd).abs()
    d_xh = C_STAT * U32 * xd.abs().amax(-1, keepdim=True) * r     # the statistics' error in xhat
    m = r * (gg + gg.mean(-1, keepdim=True) + xh.abs() * (gg * xh.abs()).mean(-1, keepdim=True))
    cond = r * d_xh * ((gg * xh.abs()).mean(-1, keepdim=True) + xh.abs() * gg.mean(-1, keepdim=True))
    err = (dx.cpu().double() - x64.grad).abs()
    bound = u * x64.grad.abs() + 2.0 ** -16 * m + cond + SUB[dtype]
    assert bool((err <= bound).all()), "dx: " + _report(err, bound)
    for name, got, ref, s, c in (("dweight", dw, w64.grad, (dyd * xh).abs().sum(0), (dyd.abs() * d_xh).sum(0)),
                                 ("dbias", db, b64.grad, dyd.abs().sum(0), 0.0)):
        err = (got.cpu().double() - ref).abs()
        bound = u * ref.abs() + 2.0 ** -16 * s + c + SUB[dtype]
        assert bool((err <= bound).all()), f"{name}: " + _report(err, bound)


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("cols", [768, 5120])
def test_rmsnorm_backward_at_massive_rows(cols, dtype):
    from oracle.mmfs import rms_norm_ref
    ops = _ops()
    rows, eps, u = 4 * 20 + 1, 1e-6, U[dtype]
    g = _gen(cols + 7 + DTYPES.index(dtype))
    x = _offset_massive_rows(rows, cols, g).to(dtype)
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(dtype)
    dy = torch.randn(rows, cols, generator=g).to(dtype)
    with torch.no_grad():
        dx, dw = ops.rmsnorm_backward(x.to(DEV), w.to(DEV), dy.to(DEV), eps)
    torch.cuda.synchronize()

    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    rms_norm_ref(x64, w64, eps).backward(dy.double())
    xd, wd, dyd = x.double(), w.double(), dy.double()
    r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    s_abs = (dyd * wd * xd).abs().sum(-1, keepdim=True)
    m = r * (dyd * wd).abs() + xd.abs() * r ** 3 * s_abs / cols
    err = (dx.cpu().double() - x64.grad).abs()
    bound = u * x64.grad.abs() + 2.0 ** -16 * m + SUB[dtype]
    assert bool((err <= bound).all()), "dx: " + _report(err, bound)
    s_w = (dyd * xd * r).abs().sum(0)
    err = (dw.cpu().double() - w64.grad).abs()
    bound = u * s_w + u * w64.grad.abs() + SUB[dtype]
    assert bool((err <= bound).all()), "dweight: " + _report(err, bound)


# --------------------------------------------------------------------------------------------------------- validation
def _bad_params(C, dtype):
    other = F32 if dtype != F32 else BF16
    full = torch.ones(2 * C, dtype=dtype, device=DEV)
    return {
        "dtype": torch.ones(C, dtype=other, device=DEV),
        "numel": torch.ones(C + 8, dtype=dtype, device=DEV),
        "strided": full[::2],
    }


@pytest.mark.parametrize("which", ["weight", "bias"])
@pytest.mark.parametrize("bad", ["dtype", "numel", "strided"])
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_layernorm_and_group_norm_refuse_mismatched_weight_or_bias(dtype, bad, which):
    """A weight / bias of another dtype (autocast-style fp32 parameters with 16-bit activations), of the wrong size or
    not contiguous would be read as C elements of x's dtype: both ops must refuse it."""
    ops = _ops()
    C = 320
    p = _bad_params(C, dtype)[bad]
    assert bad != "strided" or not p.is_contiguous()
    good = torch.ones(C, dtype=dtype, device=DEV)
    x = torch.randn(4, C, device=DEV).to(dtype)
    kw = {"weight": p, "bias": good} if which == "weight" else {"weight": good, "bias": p}
    with pytest.raises(RuntimeError, match="layernorm"):
        ops.layernorm(x, kw["weight"], kw["bias"], 1e-5)
    xg = torch.randn(2, C, 8, 8, device=DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    with pytest.raises(RuntimeError, match="group_norm_nhwc"):
        ops.group_norm_nhwc(xg, 32, kw["weight"], kw["bias"], 1e-5)
