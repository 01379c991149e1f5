"""num_launches() against the kernels one forward really runs, counted by the CUDA profiler, in every numeric mode and
on both sides of the SMPL stage's 256-pose chunking."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = {"default": {}, "fp8": {"fp8": True}, "strict": {"strict": True}}


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


@pytest.fixture(scope="module")
def engines(cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config(vit_depth=2)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    return cfg, {m: TokenHMREngine(cfg, sd, smpl, device=cuda_dev, max_batch=320, use_cuda_graph=False, **kw)
                 for m, kw in MODES.items()}


def _step_names(model):
    from tokenhmr_b200._lib import check, lib
    names = []
    for i in range(lib().thmr_engine_num_steps(model._h)):
        name = ctypes.c_char_p()
        check(lib().thmr_engine_step_info(model._h, i, ctypes.byref(name), None, None))
        names.append(name.value.decode())
    return names


@pytest.mark.parametrize("B", [3, 257])
@pytest.mark.parametrize("mode", list(MODES))
def test_num_launches_counts_the_kernels_of_a_forward(engines, mode, B):
    """B = 257 gives the SMPL stage two chunks, each with its own blend GEMM and skinning kernel.  Only the engine's
    forward is profiled (the library call TokenHMREngine.forward makes), not the module's input copy and output
    clones."""
    from torch.profiler import ProfilerActivity, profile
    from tokenhmr_b200 import synth
    cfg, models = engines
    model = models[mode]
    img = synth.make_images(B, cfg, seed=B).cuda()
    model({"img": img})                       # builds the plans (and clears the workspace's padding with memsets)
    st = model._state(B, False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model._launch(st, B)
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset"))]
    assert len(kernels) == model.num_launches(), sorted(kernels)


def test_fp8_steps_are_the_default_steps(engines):
    """The FP8 mode swaps the storage of xn and h and the GEMMs that read them, not the step list."""
    from tokenhmr_b200 import synth
    cfg, models = engines
    img = synth.make_images(3, cfg, seed=3).cuda()
    for m in ("default", "fp8"):
        models[m]({"img": img})
    assert _step_names(models["fp8"]) == _step_names(models["default"])
