"""FP8 mode, host side (no GPU): the quantisation definition (tokenhmr_b200/fp8.py) exactly, the CPU emulation's GEMM,
the ABI mirrors of the new fields, and the refusal of strict + fp8 before any CUDA work."""
import ctypes
import math
from pathlib import Path

import pytest
import torch

from tokenhmr_b200 import fp8

ROOT = Path(__file__).resolve().parent.parent


def _smallest_pow2_scale(amax: float) -> float:
    """The definition, by search: the smallest s = 2^e with amax / s <= 448 (1 for amax = 0)."""
    if amax == 0.0:
        return 1.0
    e = math.floor(math.log2(amax / 448.0)) - 2
    while amax / 2.0 ** e > 448.0:
        e += 1
    return 2.0 ** e


def test_scale_rule_edges():
    cases = [0.0, 448.0, 448.0 * 2 ** -20, 448.0 * 2 ** 7, 449.0, 447.9, 1.0, 2.0 ** -30, 3.4e38, 1e-38,
             float(torch.finfo(torch.float32).tiny)]
    got = fp8.e4m3_scale(torch.tensor(cases))
    for a, s in zip(cases, got.tolist()):
        assert s == _smallest_pow2_scale(a), (a, s)
    # amax exactly a power of two times 448: that power itself (the code 448 is representable)
    assert fp8.e4m3_scale(torch.tensor([448.0 * 2 ** -3])).item() == 2 ** -3
    # one ulp above: the next power
    above = torch.nextafter(torch.tensor([448.0 * 2 ** -3]), torch.tensor([1e9]))
    assert fp8.e4m3_scale(above).item() == 2 ** -2


def test_scale_rule_random_against_search():
    g = torch.Generator().manual_seed(0)
    amax = torch.exp(torch.empty(20000).uniform_(-60, 60, generator=g)).float()
    got = fp8.e4m3_scale(amax)
    want = torch.tensor([_smallest_pow2_scale(a) for a in amax.tolist()])
    assert torch.equal(got, want)


def _codes_by_definition(x: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    return (x.double() / s.double()).float().to(torch.float8_e4m3fn)


def test_activation_quantiser_matches_definition():
    g = torch.Generator().manual_seed(1)
    R, K = 37, 384
    x = torch.randn(R, K, generator=g) * torch.exp(torch.empty(R, 1).uniform_(-8, 8, generator=g))
    x[0, :128] = 0.0                                   # amax = 0 -> s = 1, codes 0
    x[1, :128] = 0.0
    x[1, 3] = -448.0 * 2 ** 5                          # amax exactly a power of two times 448, negative
    x[2, 128:160] *= 2.0 ** -12                        # values far below their block's amax: subnormal codes
    codes, s = fp8.quantize_rows(x)
    assert s.shape == (K // 128, R) and codes.dtype == torch.float8_e4m3fn
    for r in range(R):
        for kb in range(K // 128):
            blk = x[r, kb * 128:(kb + 1) * 128]
            sd = _smallest_pow2_scale(float(blk.abs().max()))
            assert s[kb, r].item() == sd
            assert torch.equal(codes[r, kb * 128:(kb + 1) * 128].view(torch.uint8),
                               _codes_by_definition(blk, torch.tensor(sd)).view(torch.uint8))
    assert s[0, 0].item() == 1.0 and not codes[0, :128].view(torch.uint8).any()
    assert s[0, 1].item() == 2.0 ** 5 and codes[1, 3].float().item() == -448.0
    sub = codes[2, 128:256].float().abs()
    assert ((sub > 0) & (sub < 2.0 ** -6)).any()        # e4m3 subnormals (below 2^-6) do occur
    # dequantisation is exact, the quantisation error within half an e4m3 ulp (2^-4 relative) or a subnormal step
    xd = fp8.dequantize_rows(codes, s)
    step = torch.maximum(xd.abs(), s.t().repeat_interleave(128, 1) * 2.0 ** -6) * 2.0 ** -4
    assert ((xd - x).abs() <= step).all()


def test_weight_quantiser_matches_definition():
    g = torch.Generator().manual_seed(2)
    N, K = 200, 256                                    # a partial last 128-row block
    w = 0.02 * torch.randn(N, K, generator=g)
    w[:128, 128:] *= 64.0                              # every block its own scale
    w[130, 7] = -3.5
    codes, s = fp8.quantize_weight_blocks(w)
    assert s.shape == (2, 2) and codes.shape == (N, K)
    for nb in range(2):
        for kb in range(2):
            blk = w[nb * 128:(nb + 1) * 128, kb * 128:(kb + 1) * 128]
            sd = _smallest_pow2_scale(float(blk.abs().max()))
            assert s[nb, kb].item() == sd, (nb, kb)
            assert torch.equal(codes[nb * 128:(nb + 1) * 128, kb * 128:(kb + 1) * 128].view(torch.uint8),
                               _codes_by_definition(blk, torch.tensor(sd)).view(torch.uint8))
    wd = fp8.dequantize_weight_blocks(codes, s)
    assert torch.equal(wd[130, 7], torch.tensor(-3.5))


def test_emulated_linear_is_the_promoted_block_sum():
    """The emulation's GEMM: per 128-wide k-block, the fp64 dot product of the dequantised operands rounded to fp32,
    promoted by fp32 additions; it differs from the fp64 GEMM of the same operands by at most the K / 128 fp32
    roundings of the promotion and one of the bias add (2^-24 each, relative to the running magnitude)."""
    import fp8_emulation as E
    g = torch.Generator().manual_seed(3)
    x, w, b = torch.randn(50, 640, generator=g), 0.05 * torch.randn(300, 640, generator=g), torch.randn(300, generator=g)
    y = E.fp8_linear(x, w, b)
    qa, sa = fp8.quantize_rows(x)
    qw, sw = fp8.quantize_weight_blocks(w)
    A, W = fp8.dequantize_rows(qa, sa).double(), fp8.dequantize_weight_blocks(qw, sw).double()
    ref = A @ W.t() + b.double()
    bound = (640 // 128 + 1) * 2.0 ** -24 * (A.abs() @ W.abs().t() + b.double().abs())
    assert ((y.double() - ref).abs() <= bound).all()


def test_strict_and_fp8_are_refused_before_any_cuda_work():
    from tokenhmr_b200 import synth
    from tokenhmr_b200._lib import ThmrError
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    from tokenhmr_b200.weights import PackedWeights, make_config_struct
    cfg = tiny_config(vit_depth=1)
    with pytest.raises(ThmrError, match="exclusive"):
        make_config_struct(cfg, strict=True, fp8=True)
    with pytest.raises(ThmrError, match="exclusive"):
        PackedWeights({}, cfg, torch.device("cpu"), strict=True, fp8=True)
    with pytest.raises(ThmrError, match="exclusive"):
        TokenHMREngine(cfg, synth.make_state_dict(cfg), synth.make_smpl(cfg), strict=True, fp8=True)
    assert make_config_struct(cfg, fp8=True).fp8 == 1 and make_config_struct(cfg).fp8 == 0


def test_fp8_weight_packing_on_the_host():
    """PackedWeights(fp8=True) runs the ViT's qkv / fc1 / fc2 through the block quantiser and records their scales;
    every other matrix is packed as by default (fp16)."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.weights import PackedWeights
    cfg = tiny_config(vit_depth=1)
    sd = synth.make_state_dict(cfg)
    pw = PackedWeights(sd, cfg, torch.device("cpu"), fp8=True)
    by_ptr = {t.data_ptr(): t for t in pw._keep}
    blk, bs = pw.blocks[0], pw.block_scales[0]
    for wname, sname, key in (("qkv_w", "qkv_ws", "attn.qkv"), ("fc1_w", "fc1_ws", "mlp.fc1"),
                              ("fc2_w", "fc2_ws", "mlp.fc2")):
        codes, scales = by_ptr[getattr(blk, wname)], by_ptr[getattr(bs, sname)]
        want_c, want_s = fp8.quantize_weight_blocks(sd[f"backbone.blocks.0.{key}.weight"])
        assert codes.dtype == torch.float8_e4m3fn and torch.equal(codes.view(torch.uint8), want_c.view(torch.uint8))
        assert torch.equal(scales, want_s)
    assert by_ptr[blk.proj_w].dtype == torch.float16
    assert ctypes.cast(pw.struct.block_scales_host, ctypes.c_void_p).value == ctypes.addressof(pw.block_scales)
    plain = PackedWeights(sd, cfg, torch.device("cpu"))
    assert not plain.struct.block_scales_host and plain.nbytes() > pw.nbytes()


def test_block_scales_struct_and_config_sizes_match_c(tmp_path):
    import shutil
    import subprocess
    from tokenhmr_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    pairs = [("thmr_vit_block_scales", _lib.VitBlockScales), ("thmr_config", _lib.Config),
             ("thmr_weights", _lib.Weights)]
    src = tmp_path / "sizes.c"
    body = "".join(f'  printf("%s %zu %zu\\n", "{n}", sizeof({n}), {off});\n' for n, off in (
        ("thmr_vit_block_scales", "offsetof(thmr_vit_block_scales, fc2_ws)"),
        ("thmr_config", "offsetof(thmr_config, fp8)"),
        ("thmr_weights", "offsetof(thmr_weights, block_scales_host)")))
    src.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "{ROOT / "include" / "tokenhmr_b200.h"}"\n'
                   f'int main(void) {{\n{body}  return 0;\n}}\n')
    exe = tmp_path / "sizes"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-o", str(exe), str(src)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    got = {out[i]: (int(out[i + 1]), int(out[i + 2])) for i in range(0, len(out), 3)}
    offs = {"thmr_vit_block_scales": _lib.VitBlockScales.fc2_ws.offset, "thmr_config": _lib.Config.fp8.offset,
            "thmr_weights": _lib.Weights.block_scales_host.offset}
    for name, cls in pairs:
        assert got[name] == (ctypes.sizeof(cls), offs[name]), name


def test_abi_version_counts_the_fp8_fields(built_lib):
    assert built_lib.thmr_abi_version() >= 6

