"""Host-side checks for the token head's kernel tests (no GPU): the resize map tk_seq_map (through the head-training
probe) and oracle.tokenhmr_oracle.upsample_nearest_index against ATen's nn.Upsample 'nearest', and what the hl_gemm
call-site table of tests/test_gpu_token_head_train_kernels.py claims about itself."""
import bisect

import pytest
import torch
import torch.nn.functional as F

import head_train_probe as hp
from oracle import tokenhmr_oracle as O
from test_gpu_token_head_train_kernels import SITES, _planner

TOKENIZER_PAIRS = [(160, 125), (125, 90), (90, 55), (55, 21)]   # PoseSPDecoderV1's nn.Upsample sizes


def _aten_map(lin: int, lout: int, dtype) -> list[int]:
    x = torch.arange(lin, dtype=dtype).view(1, 1, lin)
    return F.interpolate(x, size=lout, mode="nearest").view(lout).long().tolist()


def test_seq_map_matches_aten_fp32_for_every_size(built_lib):
    """Every (lin, lout) in 1..160: src is ATen's fp32 map, and lo[s] .. lo[s + 1] are exactly the positions p with
    src[p] == s, lo[lin] == lout.  The oracle's restatement gives the same map."""
    bad = []
    for lin in range(1, 161):
        for lout in range(1, 161):
            src, lo = hp.tk_seq_map(lin, lout)
            want = _aten_map(lin, lout, torch.float32)
            if src != want or O.upsample_nearest_index(lout, lin).tolist() != want:
                bad.append((lin, lout))
                continue
            # src is non-decreasing, so the positions reading s are [first p with src[p] >= s, first with > s)
            assert src == sorted(src) and lo[lin] == lout, (lin, lout)
            assert lo == [bisect.bisect_left(src, s) for s in range(lin + 1)], (lin, lout)
    assert not bad, bad[:10]


@pytest.mark.parametrize("lin,lout", [(0, 5), (5, 0), (161, 5), (5, 161), (-1, 1)])
def test_seq_map_refuses_sizes_outside_its_arrays(built_lib, lin, lout):
    with pytest.raises(RuntimeError, match="outside 1..160"):
        hp.tk_seq_map(lin, lout)


def test_tokenizer_sizes_agree_with_fp64_aten():
    """The fp64 golden and the fp64 restatement resize through ATen on fp64 input.  That gives the fp32 map at the
    four sizes the tokenizer uses, which is what makes them comparable with the kernels.  Elsewhere fp64 ATen
    differs (329 of the 25,600 pairs in 1..160; e.g. 2 -> 82 reads input 1, not 0, at p = 41): the training head
    refuses non-release tokenizer sizes, so only these four are pinned."""
    for lin, lout in TOKENIZER_PAIRS:
        assert _aten_map(lin, lout, torch.float64) == _aten_map(lin, lout, torch.float32), (lin, lout)
    assert _aten_map(2, 82, torch.float64)[41] != _aten_map(2, 82, torch.float32)[41]


def test_site_table_covers_every_planner_branch():
    """What the token head's hl_gemm call-site table claims about itself; the GPU test asserts the kernel's counts."""
    by = {s.name: s for s in SITES}
    assert len(by) == len(SITES)
    for s in SITES:
        assert s.splits == _planner(s.M, s.N, s.K, s.batch, s.partial), s.name
    # empty trailing splits, and 264 splits on one tile (exactly kSplitFloats of partials)
    s = by["mixer_norm dW B=106"]
    assert (s.orient, s.splits, s.kper, s.empty_splits, s.tiles) == ("dytx", 264, 65, 3, 1)
    assert by["mixer_norm dW B=161"].empty_splits == 1
    assert by["token MLP2 dW B=106"].empty_splits >= 1 and by["token MLP1 dW B=106"].empty_splits >= 1
    # split boundaries inside a 16-wide k-block
    for name, splits, kper in (("soft lookup Z B=1", 22, 94), ("class_pred dW B=5", 8, 100),
                               ("conv dcol 21 B=5", 5, 103), ("conv_in B=1", 11, 70)):
        assert (by[name].splits, by[name].kper) == (splits, kper), name
    # each epilogue after the reduce and direct
    for flag in ("accumulate", "gelu_out", "dgelu", "bias"):
        assert any(getattr(s, flag) and s.splits == 1 for s in SITES), flag
        assert any(getattr(s, flag) and s.splits > 1 for s in SITES), flag
    assert by["token MLP1 B=5"].splits == 2 and by["token MLP1 B=161"].splits == 1
    assert by["token MLP2 dx B=5"].splits == 2 and by["token MLP2 dx B=161"].splits == 1
    assert by["dP += dZ cb^T B=1"].splits == 2 and by["dP += dZ cb^T B=5"].splits == 1
    assert by["channel MLP2 B=5"].splits > 1 and by["res conv2 B=1"].splits > 1
    # the batched output-conv backward: A at dread + 6, rows 6 apart, images 160 apart
    s = by["out conv dcol B=5"]
    assert (s.orient, s.M, s.N, s.K, s.batch, s.sA, s.a_off) == ("dyw", 21, 1536, 6, 5, (160, 6, 1), 6)
    # mixer_trans: forward direct at >= 132 tiles, its input gradient accumulated at 16 and 2 splits
    assert by["mixer_trans B=5"].tiles >= 132 and by["mixer_trans B=5"].splits == 1
    assert by["mixer_trans dx B=5"].splits == 16 and by["mixer_trans dx B=330"].splits == 2
    assert by["mixer_trans dx B=330"].accumulate
    # splits = 1 for each of its reasons: >= 132 tiles, K < 128, no split buffer
    assert any(s.splits == 1 and s.partial and s.tiles >= 132 for s in SITES)
    assert any(s.splits == 1 and s.partial and s.K < 128 for s in SITES)
    assert any(s.splits == 1 and not s.partial for s in SITES)
