"""GPU parity of the wgmma/TMA convolution kernel, one case per layer kind, through the C ABI.

Checker: CPU fp32 torch ops on the same fp16-rounded operands (the reference's own call sites), and the
SIMT global-memory checker kernel for bisecting. Tolerance: the kernel accumulates in fp32 and rounds the
output to fp16 once, so |err| <= 1 fp16 ulp of the output magnitude (+ fp16 rounding of pre-summed weights).
"""

import ctypes

import pytest
import torch

import conv_cases
from robosat_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("i", range(len(conv_cases.default_cases(None))))
def test_conv_case_matches_cpu_reference(i, cuda_device):
    lib = _lib.load()
    case = conv_cases.default_cases(cuda_device)[i]()
    ref = case.ref()
    stream = _lib.current_stream_ptr()
    plan = ctypes.c_void_p()
    _lib.check(lib.rsb_conv_plan_create(ctypes.byref(case.desc), ctypes.byref(plan)), "plan_create")
    try:
        for _ in range(3):  # re-running the same plan must give the same answer (pipeline state resets)
            case.out.zero_()
            _lib.check(lib.rsb_conv_run(plan, stream), "conv_run")
            torch.cuda.synchronize()
            got = case.result()
            tol = 6e-3 * max(1.0, ref.abs().max().item() / 8)
            assert (got - ref).abs().max().item() <= tol, case.name
        # bisecting aid: the SIMT checker agrees with the tensor-core path to within output rounding
        tc = case.result()
        case.out.zero_()
        _lib.check(lib.rsb_conv_run_simt_check(ctypes.byref(case.desc), stream), "simt")
        torch.cuda.synchronize()
        assert (case.result() - tc).abs().max().item() <= tol
    finally:
        lib.rsb_conv_plan_destroy(plan)


@pytest.mark.parametrize("i", range(len(conv_cases.split_cases(None))))
def test_split_conv_case_matches_fp64_reference(i, cuda_device):
    """Strict precision (hi/lo fp16 operand planes, 3 MMAs per K step, fp32 accumulate in registers) against a float64
    reference of the same operation on the values the planes represent. Tolerance: 2e-5 of the output range. (The tensor
    core's fp32 accumulation is not round-to-nearest, so its error grows with the length of one accumulation chain; the plan
    cuts long K loops into chunks that the epilogue adds in round-to-nearest fp32 -- rsb_conv_desc.kchunk.)"""
    lib = _lib.load()
    case = conv_cases.split_cases(cuda_device)[i]()
    ref = case.ref()
    stream = _lib.current_stream_ptr()
    plan = ctypes.c_void_p()
    _lib.check(lib.rsb_conv_plan_create(ctypes.byref(case.desc), ctypes.byref(plan)), "plan_create")
    try:
        outs = []
        for _ in range(2):
            case.out.zero_()
            _lib.check(lib.rsb_conv_run(plan, stream), "conv_run")
            torch.cuda.synchronize()
            outs.append(case.out.clone())
        assert torch.equal(outs[0], outs[1]), "split conv is not deterministic"
        got = case.result()
        scale = max(1.0, ref.abs().max().item())
        err = (got - ref).abs().max().item()
        print("%s: max|err| %.3e (%.2e of range)" % (case.name, err, err / scale))
        assert err <= 2e-5 * scale, (case.name, err)
        # the SIMT checker (plain fp32 FMAs on hi + lo) agrees
        case.out.zero_()
        _lib.check(lib.rsb_conv_run_simt_check(ctypes.byref(case.desc), stream), "simt")
        torch.cuda.synchronize()
        assert (case.result() - got).abs().max().item() <= 4e-5 * scale
    finally:
        lib.rsb_conv_plan_destroy(plan)


def test_split_prepass_and_maxpool(cuda_device):
    """strict-precision helpers: the pre-pass writes half(x) and half(x - half(x)); the max pool of pairs == max of the sums"""
    import emulate
    from robosat_b200 import synth

    lib = _lib.load()
    u8 = synth.make_tiles_u8(2, 64, seed=5)
    ref = emulate.prepass_s2d_split_cpu(synth.normalize_tiles(u8))
    dst = torch.zeros(2, 2, 32, 36, 16, dtype=torch.float16, device=cuda_device)
    mean = (ctypes.c_float * 3)(*synth.IMAGENET_MEAN)
    std = (ctypes.c_float * 3)(*synth.IMAGENET_STD)
    u8d = u8.to(cuda_device)
    _lib.check(lib.rsb_prepass_s2d_split(u8d.data_ptr(), 1, dst.data_ptr(), dst.numel() // 2, 2, 64, 64, mean, std, _lib.current_stream_ptr()), "prepass")
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), ref)
    g = torch.Generator().manual_seed(3)
    for (N, H, W, C, k, s, p) in [(2, 32, 32, 64, 3, 2, 1), (3, 8, 8, 2048, 2, 2, 0)]:
        x = torch.randn((N, C, H, W), generator=g)
        hi = x.half()
        lo = (x - hi.float()).half()
        val = hi.float() + lo.float()
        ref = torch.nn.functional.max_pool2d(val, k, s, p)
        src = torch.stack([hi, lo]).permute(0, 1, 3, 4, 2).contiguous().to(cuda_device)
        dst = torch.zeros(2, N, ref.shape[2], ref.shape[3], C, dtype=torch.float16, device=cuda_device)
        _lib.check(lib.rsb_maxpool_nhwc_split(src.data_ptr(), src.numel() // 2, dst.data_ptr(), dst.numel() // 2, N, H, W, C, k, s, p,
                                              _lib.current_stream_ptr()), "maxpool_split")
        torch.cuda.synchronize()
        d = dst.cpu()
        assert torch.equal((d[0].float() + d[1].float()).permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize("block_n", [64, 128, 256])
def test_conv_multi_wave_persistent_schedule(block_n, cuda_device):
    """More tiles than SMs: every CTA loops over several tiles and every pipeline stage is reused across tiles."""
    lib = _lib.load()
    case = conv_cases.conv_case("3x3", 8, 64, 64, 64, 256, cuda_device, seed=21, block_n=block_n)
    plan = ctypes.c_void_p()
    _lib.check(lib.rsb_conv_plan_create(ctypes.byref(case.desc), ctypes.byref(plan)), "plan_create")
    _lib.check(lib.rsb_conv_run(plan, _lib.current_stream_ptr()), "conv_run")
    torch.cuda.synchronize()
    ref = case.ref()
    assert (case.result() - ref).abs().max().item() <= 6e-3 * max(1.0, ref.abs().max().item() / 8)
    lib.rsb_conv_plan_destroy(plan)


_PAIR_CASES = [
    lambda d: conv_cases.conv_case("1x1", 1, 16, 32, 256, 128, d, seed=2, residual=True, block_n=128),
    lambda d: conv_cases.conv_case("3x3", 1, 24, 40, 128, 256, d, seed=4, block_n=256),
    lambda d: conv_cases.conv_case("3x3", 8, 64, 64, 64, 256, d, seed=21, block_n=128),   # multi-wave
    lambda d: conv_cases.conv_case("3x3", 5, 8, 8, 128, 256, d, seed=22, block_n=256),    # odd number of spatial tiles
    lambda d: conv_cases.conv_case("1x1", 3, 8, 8, 512, 2048, d, seed=7, residual=True, block_n=256),
    lambda d: conv_cases.conv_case("3x3s2", 2, 32, 32, 128, 128, d, seed=5, block_n=128),
    lambda d: conv_cases.decoder_case(3, 4, 4, [256, 256], 256, d, seed=10, block_n=128),
]


@pytest.mark.parametrize("i", range(len(_PAIR_CASES)))
def test_conv_cta_pair_matches_single_cta(i, cuda_device):
    """CTA-pair schedule (a cluster of two CTAs on neighbouring tiles, each loading half of the shared weight tile and multicasting it) == one CTA per tile, bit for bit."""
    lib = _lib.load()
    case = _PAIR_CASES[i](cuda_device)
    stream = _lib.current_stream_ptr()
    outs = []
    for pair in (0, 1):
        case.desc.cta_pair = pair
        plan = ctypes.c_void_p()
        _lib.check(lib.rsb_conv_plan_create(ctypes.byref(case.desc), ctypes.byref(plan)), "plan_create")
        try:
            for _ in range(2):
                case.out.zero_()
                _lib.check(lib.rsb_conv_run(plan, stream), "conv_run")
                torch.cuda.synchronize()
            outs.append(case.out.clone())
        finally:
            lib.rsb_conv_plan_destroy(plan)
    ref = case.ref()
    assert (case.result() - ref).abs().max().item() <= 6e-3 * max(1.0, ref.abs().max().item() / 8), case.name
    assert torch.equal(outs[0], outs[1]), case.name


def test_prepass_u8_matches_reference_transform(cuda_device):
    """uint8 NHWC -> normalised fp16 s2d == ToTensor + Normalize (predict.py:71-73) then fp16 rounding."""
    import emulate
    from robosat_b200 import synth

    lib = _lib.load()
    u8 = synth.make_tiles_u8(2, 64, seed=5)
    ref = emulate.prepass_s2d_cpu(synth.normalize_tiles(u8))
    dst = torch.zeros(2, 32, 36, 16, dtype=torch.float16, device=cuda_device)
    mean = (ctypes.c_float * 3)(*synth.IMAGENET_MEAN)
    std = (ctypes.c_float * 3)(*synth.IMAGENET_STD)
    u8d = u8.to(cuda_device)
    _lib.check(lib.rsb_prepass_s2d(u8d.data_ptr(), 1, dst.data_ptr(), 2, 64, 64, mean, std, _lib.current_stream_ptr()), "prepass")
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), ref)


def test_maxpool_matches_torch(cuda_device):
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    for (N, H, W, C, k, s, p) in [(2, 32, 32, 64, 3, 2, 1), (3, 8, 8, 2048, 2, 2, 0)]:
        x = torch.randn((N, C, H, W), generator=g).half()
        ref = torch.nn.functional.max_pool2d(x.float(), k, s, p).half()
        src = x.permute(0, 2, 3, 1).contiguous().to(cuda_device)
        dst = torch.zeros(N, ref.shape[2], ref.shape[3], C, dtype=torch.float16, device=cuda_device)
        _lib.check(lib.rsb_maxpool_nhwc(src.data_ptr(), dst.data_ptr(), N, H, W, C, k, s, p, _lib.current_stream_ptr()), "maxpool")
        torch.cuda.synchronize()
        assert torch.equal(dst.cpu().permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize("i", range(len(conv_cases.row_cases(None))))
def test_row_conv_case_matches_cpu_reference(i, cuda_device):
    """line-buffer kernel (shared-memory row ring, shifted operand windows) against the same CPU references"""
    from robosat_b200.engine import RowConvOp

    case = conv_cases.row_cases(cuda_device)[i]()
    ref = case.ref()
    op = RowConvOp(case.name, case.desc)
    tol = 6e-3 * max(1.0, ref.abs().max().item() / 8)
    for _ in range(2):
        case.out.zero_()
        op.run(_lib.current_stream_ptr())
        torch.cuda.synchronize()
        assert (case.result() - ref).abs().max().item() <= tol, case.name


@pytest.mark.parametrize("i", range(len(conv_cases.row_split_cases(None))))
def test_row_split_case_matches_fp64_reference(i, cuda_device):
    """strict-precision line-buffer kernel (dec5 + final): hi/lo row ring, [W_hi | W_lo] in one MMA + A_lo W_hi in a second"""
    from robosat_b200.engine import RowConvOp

    case = conv_cases.row_split_cases(cuda_device)[i]()
    ref = case.ref()
    op = RowConvOp(case.name, case.desc)
    scale = max(1.0, ref.abs().max().item())
    for _ in range(2):
        case.out.zero_()
        op.run(_lib.current_stream_ptr())
        torch.cuda.synchronize()
        err = (case.result() - ref).abs().max().item()
        print("%s: max|err| %.3e (%.2e of range)" % (case.name, err, err / scale))
        assert err <= 1e-5 * scale, case.name


@pytest.mark.parametrize("kind,N,H,W,cin,cout,block_n,pair", [
    ("1x1", 2, 24, 40, 64, 64, 32, 0),      # ragged tiles (W, H not multiples of the tile box), 32-column chunks
    ("1x1", 3, 16, 16, 64, 256, 64, 0),
    ("3x3", 2, 20, 36, 64, 128, 128, 0),    # 8 epilogue warps (two per lane quarter)
    ("3x3s2", 2, 32, 32, 128, 256, 256, 0),
    ("3x3", 4, 16, 16, 128, 256, 128, 1),   # CTA pair
    ("1x1", 3, 24, 16, 256, 512, 256, 1),   # CTA pair, odd number of spatial tiles (last pair half empty)
])
def test_conv_stats_epilogue_partials_fold_to_float64_batchnorm(kind, N, H, W, cin, cout, block_n, pair, cuda_device):
    """rsb_conv_desc.stats: the per-quarter-tile column sums of the fp16 outputs, written by the conv epilogue, fold to the
    float64 BatchNorm batch statistics of the stored z: same mean / invstd / scale / shift / running statistics to fp32
    rounding; the conv output itself is bit-identical to the plain instance."""
    lib = _lib.load()
    stream = _lib.current_stream_ptr()
    case = conv_cases.conv_case(kind, N, H, W, cin, cout, cuda_device, seed=11, relu=False, bias=False, block_n=block_n, cta_pair=bool(pair))
    d = case.desc
    plan = ctypes.c_void_p()
    _lib.check(lib.rsb_conv_plan_create(ctypes.byref(d), ctypes.byref(plan)), "plan_create")
    _lib.check(lib.rsb_conv_run(plan, stream), "conv_run")
    torch.cuda.synchronize()
    plain = case.out.clone()
    lib.rsb_conv_plan_destroy(plan)

    rows = 4 * (-(-d.Wt // d.TW)) * (-(-d.Ht // d.TH)) * (-(-d.Nt // d.TN))
    partials = torch.full((rows, 2, cout), float("nan"), dtype=torch.float32, device=cuda_device)
    d.stats, d.stats_bytes = partials.data_ptr(), partials.numel() * 4
    _lib.check(lib.rsb_conv_plan_create(ctypes.byref(d), ctypes.byref(plan)), "plan_create(stats)")
    try:
        case.out.zero_()
        _lib.check(lib.rsb_conv_run(plan, stream), "conv_run(stats)")
        torch.cuda.synchronize()
        assert torch.equal(case.out, plain)
        assert torch.isfinite(partials).all(), "a partial entry was not written"
        z = case.out.reshape(-1, cout).double()
        M = z.shape[0]
        tot = partials.double().sum(0)
        assert torch.allclose(tot[0], z.sum(0), rtol=1e-5, atol=1e-3)
        assert torch.allclose(tot[1], (z * z).sum(0), rtol=1e-5, atol=1e-3)

        g = torch.Generator().manual_seed(3)
        ga = (torch.rand(cout, generator=g) + 0.5).to(cuda_device)
        be = torch.randn(cout, generator=g).to(cuda_device)
        rm, rv = torch.zeros(cout, device=cuda_device), torch.ones(cout, device=cuda_device)
        nb = torch.zeros(1, dtype=torch.int64, device=cuda_device)
        o1 = [torch.empty(cout, device=cuda_device) for _ in range(4)]
        sums = torch.zeros(20 * cout, dtype=torch.float64, device=cuda_device)
        for _ in range(3):  # the accumulators are left clean for the next call
            _lib.check(lib.rsb_bn_partials_finalize(partials.data_ptr(), rows, sums.data_ptr(), ga.data_ptr(), be.data_ptr(), rm.data_ptr(),
                                                    rv.data_ptr(), nb.data_ptr(), *[t.data_ptr() for t in o1], M, cout, 1e-5, 0.1, stream),
                       "partials_finalize")
        torch.cuda.synchronize()
        assert int(nb) == 3
        # float64 reference: biased variance for the normalisation, the unbiased one for the running update (momentum 0.1)
        mean = z.sum(0) / M
        var = ((z * z).sum(0) / M - mean * mean).clamp_min(0)
        invstd = 1.0 / torch.sqrt(var + 1e-5)
        scale = ga.double() * invstd
        shift = be.double() - mean * scale
        rm_ref, rv_ref = torch.zeros_like(mean), torch.ones_like(mean)
        for _ in range(3):
            rm_ref = 0.9 * rm_ref + 0.1 * mean
            rv_ref = 0.9 * rv_ref + 0.1 * var * M / (M - 1)
        for got, want in zip(o1 + [rm, rv], [mean, invstd, scale, shift, rm_ref, rv_ref]):
            assert torch.allclose(got.double(), want, rtol=2e-5, atol=2e-6), (got.double() - want).abs().max()
    finally:
        lib.rsb_conv_plan_destroy(plan)


def test_conv_stats_rejects_unsupported_descriptors(cuda_device):
    lib = _lib.load()
    case = conv_cases.conv_case("1x1", 1, 16, 16, 64, 64, cuda_device, relu=False, bias=False, residual=True)
    buf = torch.zeros(1 << 16, dtype=torch.float32, device=cuda_device)
    case.desc.stats, case.desc.stats_bytes = buf.data_ptr(), buf.numel() * 4
    plan = ctypes.c_void_p()
    assert lib.rsb_conv_plan_create(ctypes.byref(case.desc), ctypes.byref(plan)) == -1      # residual
    case = conv_cases.conv_case("1x1", 1, 16, 16, 64, 64, cuda_device, relu=False, bias=False)
    case.desc.stats, case.desc.stats_bytes = buf.data_ptr(), 64
    assert lib.rsb_conv_plan_create(ctypes.byref(case.desc), ctypes.byref(plan)) == -1      # buffer too small
