"""Per-element kernel contract of include/yume_b200_clip.h (`-m gpu`): yb_resize_bicubic_normalize against an fp64 reference
computed on the device from the same fp32 input, with the bound derived below, on a NaN-poisoned output between guard planes,
and against PyTorch's own F.interpolate + Normalize on the same device (bit-exact at the identity size; elsewhere the number
of differing elements and the largest difference are reported).

Machinery (Guarded / guarded / assert_within / _gen) is that of tests/test_gpu_kernel_contract.py. The helpers above the
fixtures need no GPU; tests/test_clip_cpu.py runs them on the CPU, including the defects the bound must reject (an unclamped
tap, align_corners=True, an antialiased resample). u32 = 2^-24.
"""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernel_contract import U32, _gen, assert_within, guarded, record_exact

pytestmark = pytest.mark.gpu

MEAN = (0.48145466, 0.4578275, 0.40821073)      # OpenAI CLIP (wan/modules/clip.py:457-458)
STD = (0.26862954, 0.26130258, 0.27577711)
RESIZE_SIZES = [(544, 960), (224, 224), (150, 200), (33, 47), (480, 832), (720, 1280)]
COEF_ERR = 256 * U32            # |fp32 Keys coefficient - exact coefficient of the same t| (derivation: resize_bound)
COEF_ABS_SUM = 1.5              # max over t of sum_k |W(t + 1 - k)| for A = -0.75 (1.375 at t = 0.5; checked on the CPU)


# ------------------------------------------------------------------------------------------------------------
# reference and bound (no GPU needed)
# ------------------------------------------------------------------------------------------------------------
def source_coords(n_in, n_out, align_corners=False, device="cpu"):
    """The kernel's source coordinate per output index: scale = fp32(n_in / n_out), src = fp32(scale * (d + 0.5) - 0.5) with
    ONE rounding (the product and difference are exact in fp64, then rounded to fp32 = fmaf). Returns (floor, t) with t in
    [0, 1) in fp64; t = src - floor(src) is exact in fp32. align_corners=True (a defect here): scale = (n_in-1)/(n_out-1),
    src = scale * d."""
    d = torch.arange(n_out, dtype=torch.float64, device=device)
    if align_corners:
        scale = torch.tensor((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0, dtype=torch.float32).double()
        src = (scale * d).float().double()
    else:
        scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
        src = (scale.double().to(device) * (d + 0.5) - 0.5).float().double()
    fl = torch.floor(src)
    return fl.long(), src - fl


def keys_weights(t, A=-0.75):
    """[n, 4] Keys cubic weights of taps floor-1 .. floor+2 at fractional offset t (fp64)."""
    def w1(x):
        return ((A + 2) * x - (A + 3)) * x * x + 1

    def w2(x):
        return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A
    return torch.stack([w2(t + 1), w1(t), w1(1 - t), w2(2 - t)], dim=-1)


def _taps(fl, n_in):
    idx = fl[:, None] + torch.arange(-1, 3, device=fl.device)[None, :]
    valid = (idx >= 0) & (idx < n_in)
    return idx.clamp(0, n_in - 1), valid


def resize_ref(x, S, mean=MEAN, std=STD, clamp=True, align_corners=False):
    """fp64 reference of yb_resize_bicubic_normalize from the fp32 image x [C, H, W]: the kernel's fp32 source coordinates
    (source_coords), exact Keys weights, border-clamped taps (clamp=False reads zero outside: a defect), then
    (v * 0.5 + 0.5 - mean) / std exactly. H == W == S copies. Returns (out [C, S, S], interpolated v [C, S, S],
    tap magnitude M [S, S] = max |x| over the 16 taps of each output pixel, over channels)."""
    C, H, W = x.shape
    xd = x.double()
    if H == S and W == S and not align_corners:
        v = xd.clone()
        M = xd.abs().amax(dim=0)
    else:
        fy, ty = source_coords(H, S, align_corners, x.device)
        fx, tx = source_coords(W, S, align_corners, x.device)
        iy, vy = _taps(fy, H)
        ix, vx = _taps(fx, W)
        wy, wx = keys_weights(ty), keys_weights(tx)
        if not clamp:
            wy, wx = wy * vy, wx * vx
        g = xd[:, iy[:, :, None, None], ix[None, None, :, :]]          # [C, S, 4, S, 4]
        v = torch.einsum("cyaxb,ya,xb->cyx", g, wy, wx)
        M = g.abs().amax(dim=(0, 2, 4))
    m = torch.tensor(mean, dtype=torch.float32, device=x.device).double().view(-1, 1, 1)
    s = torch.tensor(std, dtype=torch.float32, device=x.device).double().view(-1, 1, 1)
    return (v * 0.5 + 0.5 - m) / s, v, M


def resize_bound(x, S, out_ref, v_ref, M, mean=MEAN, std=STD):
    """Per-element bound of the kernel against resize_ref.
    Coefficients: each Keys weight is a cubic evaluated in fp32 (Horner form, <= 6 roundings) at x in [0, 2]; Higham's Horner
    bound gives gamma_6 * sum_i |a_i| |x|^i <= 6.0001 u32 * 36 (A = -0.75, worst at x = 2) = 216 u32, and rounding t + 1 / 1 - t
    moves x by <= 2 u32 with |W'| <= 1.35: COEF_ERR = 256 u32 covers both.
    Interpolation, with M = max |x| over the 16 taps and sum |c| <= 1.5 (COEF_ABS_SUM; 1.51 with the coefficient errors):
    each row r_k = sum_j c_j x_kj takes <= 4 roundings, |dr_k| <= 4*COEF_ERR*M + 4 u32 * 1.51 M; the column pass adds
    4*COEF_ERR*1.51 M (coefficients) + 1.51 max|dr_k| + 4 u32 * 1.51^2 M (roundings):
      E_v <= (12.08 * COEF_ERR + 18.3 u32) M = 3111 u32 * M, taken as 3200 u32 * M.
    Normalize: w = v*0.5 + 0.5, w - mean and the IEEE divide round once each (<= u32 of each magnitude), so
      |out - ref| <= (0.5 E_v + u32 (|w| + |w - mean|)) / std + u32 |out|, taken with factor 2 on the rounding terms.
    The identity size copies: E_v = 0."""
    C, H, W = x.shape
    s = torch.tensor(std, dtype=torch.float32, device=x.device).double().view(-1, 1, 1)
    m = torch.tensor(mean, dtype=torch.float32, device=x.device).double().view(-1, 1, 1)
    w = v_ref * 0.5 + 0.5
    Ev = torch.zeros_like(M) if (H == S and W == S) else 3200 * U32 * M
    return (0.5 * Ev + 2 * U32 * (w.abs() + (w - m).abs())) / s + 2 * U32 * out_ref.abs()


def strided_image(g, H, W, device):
    """An fp32 [3, 1, H, W] image in [-1, 1] as a strided view of a channels-last [H + 3, W + 5, 3] buffer (the resize reads
    it in place), plus a few values just inside [-1, 1] at the borders, where clamping matters."""
    full = torch.rand(H + 3, W + 5, 3, generator=g) * 2 - 1
    full[1, 2:2 + W] = 0.999
    full[1:1 + H, 2] = -0.999
    return full.to(device)[1:1 + H, 2:2 + W].permute(2, 0, 1)[:, None]


# ------------------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


@pytest.mark.parametrize("H,W", RESIZE_SIZES)
def test_resize_bicubic_normalize_per_element(dev, H, W):
    """The CLIP preprocessing on the image sizes the I2V pipeline feeds it (480x832, 544x960, 720x1280), the identity size,
    an upscale and an odd size. fp64 reference and bound: resize_ref / resize_bound. The output is a NaN-poisoned [3, 224, 224]
    between two guard planes; the input a strided channels-last view. Also compared with F.interpolate + Normalize on the
    device: bit-exact at 224x224 (the reference copies), elsewhere the differing elements are reported."""
    from yume_b200 import ops
    S = 224
    g = _gen("resize_bicubic_normalize", H, W)
    img = strided_image(g, H, W, dev)
    mean = torch.tensor(MEAN, dtype=torch.float32, device=dev)
    std = torch.tensor(STD, dtype=torch.float32, device=dev)
    out = guarded((3, S, S), torch.float32, pad=(1, 0))
    ops.resize_bicubic_normalize(img[:, 0], out.view, mean, std)
    torch.cuda.synchronize()
    tag = f"resize {H}x{W} -> {S}"
    out.check(tag)
    ref, v, M = resize_ref(img[:, 0], S)
    assert_within(out.view, ref, resize_bound(img[:, 0], S, ref, v, M), tag, "resize_bicubic_normalize")

    tv = F.interpolate(img.transpose(0, 1), size=(S, S), mode="bicubic", align_corners=False)
    tv = tv.mul_(0.5).add_(0.5).sub_(mean.view(-1, 1, 1)).div_(std.view(-1, 1, 1))[0]
    diff = (out.view != tv)
    if (H, W) == (S, S):
        assert not diff.any(), f"{tag}: {int(diff.sum())} elements differ from F.interpolate + Normalize"
        record_exact("resize_bicubic_normalize identity")
    n = int(diff.sum())
    print(f"[contract] {tag}: {n} of {diff.numel()} elements differ from F.interpolate + Normalize on this device "
          f"(max |diff| {float((out.view - tv).abs().max()):.3g})")


def test_resize_bicubic_normalize_rejects_bad_arguments(dev):
    from yume_b200 import _lib
    lib = _lib.load()
    assert lib.yb_resize_bicubic_normalize(None, 1, 1, 1, 3, 4, 4, None, 4, None, None, None) == -1    # YB_ERR_ARG
    x = torch.zeros(3, 4, 4, device=dev)
    assert lib.yb_resize_bicubic_normalize(x.data_ptr(), 16, 4, 1, 3, 0, 4, x.data_ptr(), 4, x.data_ptr(), x.data_ptr(),
                                           None) == -1


# entry point -> tests that exercise it (tests/test_clip_cpu.py applies the entry-point guard to include/yume_b200_clip.h)
COVERS = {
    "yb_resize_bicubic_normalize": ["test_resize_bicubic_normalize_per_element",
                                    "test_resize_bicubic_normalize_rejects_bad_arguments"],
}
