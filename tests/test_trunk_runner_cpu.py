"""CPU (dry device): a trunk runner refuses a pass it cannot run before it launches anything.  Its buffers are sized for N
images, and every kernel of a pass indexes pix, the plan and feats by the pass's own n: a pass of more images than the runner
holds, or tensors of the wrong type, shape, layout or device, would write past the runner's buffers or read garbage.  A valid
16-bit pass is still the eleven launches of trunk_bf16.forward."""
import ctypes as C

import numpy as np
import pytest
import torch

N = 8
ELEVEN = ["serl_trunk_stem_prep_h16", "serl_stem_conv_pool_tc_h16", "serl_pool_finish_gn_h16", "serl_conv3x3_res_h16", "serl_conv3x3_res_h16",
          "serl_conv3x3s2_res_h16", "serl_conv3x3_res_h16", "serl_conv3x3s2_res_h16", "serl_conv3x3_res_h16", "serl_conv3x3s2_res_h16",
          "serl_conv3x3_res_h16"]


@pytest.fixture()
def dry(monkeypatch):
    """Kernel launches replaced by a recorder of (entry point, weight addresses its descriptor names)."""
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        d = args[0]._obj if args and isinstance(args[0], type(C.byref(C.c_int()))) else None
        calls.append((name, tuple(getattr(d, f) for f in ("w", "w_proj") if getattr(d, f, None))))
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(L, "new_event", lambda: Ev())
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: len(calls))
    return calls


def _runner(precision, n=N):
    from serl_b200.params import init_trunk
    from serl_b200.trunk import FrozenTrunk
    w = {k: torch.as_tensor(v) for k, v in init_trunk(np.random.default_rng(0)).items()}
    return FrozenTrunk({"cam": w}, precision).runner(n, "cpu")


def _pix(n, hw=128, c=3, dtype=torch.uint8):
    return torch.zeros(n, hw, hw, c, dtype=dtype)


def _feats(n, dtype=torch.float32):
    return torch.zeros(n, 4, 4, 512, dtype=dtype)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("n", [1, 5, N])
def test_a_valid_16bit_pass_is_the_eleven_launches(dry, precision, n):
    r = _runner(precision)
    r.forward("cam", _pix(n), _feats(N))
    assert [name for name, _ in dry] == ELEVEN


def test_a_valid_fp32_pass_launches(dry):
    r = _runner("fp32")
    r.forward("cam", _pix(3), _feats(3))
    assert len(dry) > 0 and all(name.endswith("_f32") for name, _ in dry)


def _bad_passes():
    """(label, pix, feats) of passes a runner for N images must refuse."""
    feats = _feats(N)
    return [
        ("n > N", _pix(N + 1), _feats(N + 1)),
        ("n = 0", _pix(0), feats),
        ("64x64 frames", _pix(N, 64), feats),
        ("256x256 frames", _pix(N, 256), feats),
        ("4 channels", _pix(N, c=4), feats),
        ("float pix", _pix(N, dtype=torch.float32), feats),
        ("3-d pix", _pix(N)[0], feats),
        ("strided pix", torch.zeros(N, 128, 128, 6, dtype=torch.uint8)[..., :3], feats),
        ("pix not on the runner's device", _pix(N).to("meta"), feats),
        ("fewer feature rows than images", _pix(N), _feats(N - 1)),
        ("fp16 feats", _pix(N), _feats(N, torch.float16)),
        ("flat feats", _pix(N), torch.zeros(N, 4 * 4 * 512)),
        ("feats of the wrong width", _pix(N), torch.zeros(N, 4, 4, 256)),
        ("strided feats", _pix(N), torch.zeros(2 * N, 4, 4, 512)[::2]),
        ("feats not on the runner's device", _pix(N), feats.to("meta")),
    ]


@pytest.mark.parametrize("precision", ["fp16", "bf16", "fp32"])
@pytest.mark.parametrize("case", range(len(_bad_passes())), ids=[c[0] for c in _bad_passes()])
def test_a_runner_refuses_a_bad_pass_before_any_launch(dry, precision, case):
    label, pix, feats = _bad_passes()[case]
    r = _runner(precision)
    with pytest.raises(ValueError, match="trunk pass"):
        r.forward("cam", pix, feats)
    assert dry == [], label
    assert not r.plans and r._f32 is None                           # nothing was allocated for the refused pass either


def test_a_smaller_pass_after_a_full_one_is_accepted(dry):
    r = _runner("fp16")
    r.forward("cam", _pix(N), _feats(N))
    r.forward("cam", _pix(1), _feats(N))
    assert [name for name, _ in dry] == ELEVEN + ELEVEN


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_a_plan_refuses_a_pass_larger_than_itself(dry, precision):
    """Kernel tests and callers that build plans directly go through trunk_bf16.forward alone: it checks n against the plan."""
    from serl_b200 import trunk_bf16 as T
    from serl_b200.params import init_trunk
    w = {k: torch.as_tensor(v) for k, v in init_trunk(np.random.default_rng(0)).items()}
    wp = T.pack_trunk(w, T.FMT[precision][1])
    plan = T._Plan(4, 128, "cpu", precision)
    assert plan.N == 4
    for n in (5, 0):
        with pytest.raises(ValueError, match="trunk pass"):
            T.forward(plan, w, wp, _pix(n), _feats(max(n, 1)))
        assert dry == []
    T.forward(plan, w, wp, _pix(4), _feats(4))
    assert [name for name, _ in dry] == ELEVEN


def test_resident_units_refuses_unknown_launches_and_formats():
    """serl_trunk_resident_units answers only for the trunk's eight persistent launches and the two 16-bit formats; anything else
    is refused on the host, before any device query."""
    from serl_b200 import _lib as L
    lib = L.load()
    assert lib.serl_trunk_resident_units(L.TRUNK_RES4 + 1, L.FMT_FP16) < 0
    assert lib.serl_trunk_resident_units(-1, L.FMT_BF16) < 0
    assert lib.serl_trunk_resident_units(L.TRUNK_STEM, 7) < 0
    assert b"serl_trunk_resident_units" in lib.serl_last_error()
