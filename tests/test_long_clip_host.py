"""CPU checks of the inputs beyond the pipeline's own shapes: UNetVideoModel.forward on more than 8 frames and Propagation
with flows at another resolution or temporal length than the latents.

The oracle is pinned to fixtures minted from the unmodified reference (oracle/make_golden_long.py): the log-bucket and
saturated relative-position biases and the area resize of the flows.  The host logic then runs against the same fixtures
with the emulated kernels of tests/emu_ops.py, plus a torch stand-in for the flow resize defined here."""
import ctypes as C
import json
import os
import zlib

import pytest
import torch
import torch.nn.functional as F

import emu_ops
from oracle import uav_oracle as O
from oracle.weights import make_state_dict

G = os.path.join(os.path.dirname(__file__), "golden")
CFG = os.path.join(os.path.dirname(__file__), "..", "upscale_a_video_b200", "configs")
META = json.load(open(os.path.join(G, "meta.json")))
PROP_MODES = (("nearest", "fuse", 0.001, 0.05), ("bilinear", "copy", 0.01, 0.5))


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def _load(name):
    return torch.load(os.path.join(G, name), map_location="cpu", weights_only=False)


def _unet_long_case(name):
    """a case of unet_long.pt with its inputs redrawn: sample, low_res and the text embeddings are drawn in that order from a
    generator seeded with crc32(name) (oracle/make_golden_long.py); the stored sums catch a change of torch's generator"""
    c = dict(_load("unet_long.pt")[name])
    B, T, H, W = c["shape"]
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    c["sample"] = torch.randn(B, 4, T, H, W, generator=g)
    c["low_res"] = torch.randn(B, 3, T, H, W, generator=g)
    c["ctx"] = torch.randn(B, 77, 1024, generator=g) * 0.3
    for k, want in zip(("sample", "low_res", "ctx"), c["input_sums"]):
        assert abs(float(c[k].double().sum()) - want) < 1e-6 * (1 + abs(want)), f"{name}: redrawn {k} differs from the fixture's"
    return c


def _ucfg():
    return json.load(open(os.path.join(CFG, "unet_video_config.json")))


@pytest.fixture(scope="module")
def unet_sd():
    shapes = json.load(open(os.path.join(G, "shapes_unet.json")))
    return make_state_dict(shapes, META["seed_unet"])


def flow_resize_area_standin(flows, size, scale):
    """what ops.flow_resize_area computes: F.interpolate(mode='area') * scale in the flows' dtype"""
    return F.interpolate(flows, tuple(size), mode="area") * scale


@pytest.fixture()
def emulated(monkeypatch):
    from upscale_a_video_b200 import _lib, layers, propagation_module, unet_video
    monkeypatch.setattr(emu_ops, "flow_resize_area", flow_resize_area_standin, raising=False)
    for mod in (layers, unet_video, propagation_module):
        monkeypatch.setattr(mod, "ops", emu_ops)
    monkeypatch.setattr(_lib, "require_cuda", lambda t, who: None)


# ------------------------------------------------------------------ oracle vs the reference's fixtures
@pytest.mark.parametrize("case", ["t12_16x24", "t40_8x8"])
def test_oracle_unet_long_clip(unet_sd, case):
    c = _unet_long_case(case)
    with torch.no_grad():
        out = O.unet_forward(unet_sd, _ucfg(), c["sample"], torch.tensor(c["timestep"]), c["low_res"], c["ctx"],
                             c["class_labels"])
    torch.testing.assert_close(out, c["out"], rtol=1e-4, atol=1e-4)


def test_oracle_propagation_resized_flows():
    p = _load("propagation_resize.pt")
    x = p["x"]
    assert set(p) == {"x", "up2x", "down2x", "ratio1_5", "t7"}
    for name in ("up2x", "down2x", "ratio1_5", "t7"):
        c = p[name]
        assert tuple(c["flows_forward"].shape[2:]) != (x.shape[2] - 1, *x.shape[3:])
        for dt in (torch.float32, torch.float16):
            for interp, mode, a1, a2 in PROP_MODES:
                out = O.propagation(x.to(dt), c["flows_forward"].to(dt), c["flows_backward"].to(dt), interp, mode, 0.5, a1, a2)
                assert torch.equal(out, c[f"{str(dt)[6:]}/{interp}_{mode}"]), (name, dt, interp)


def test_relative_position_bias_table_matches_oracle():
    """exact buckets below distance 8, log buckets from 8 to 32, the saturated buckets 15 / 31 beyond"""
    from upscale_a_video_b200.layers import RelativePositionBias
    rpb = RelativePositionBias(heads=8, max_distance=32)
    with torch.no_grad():
        rpb.relative_attention_bias.weight.copy_(torch.randn(32, 8, generator=torch.Generator().manual_seed(4)))
    sd = {"b.relative_attention_bias.weight": rpb.relative_attention_bias.weight.detach()}
    for n in range(1, 65):
        assert torch.equal(rpb.table(n), O.rel_pos_bias(sd, "b", n)), n
    # distance 40 uses the saturated bucket of its direction: 31 for keys after the query, 15 for keys before it
    t = rpb.table(64)
    w = rpb.relative_attention_bias.weight.detach()
    assert torch.equal(t[:, 0, 40], w[31]) and torch.equal(t[:, 40, 0], w[15])


# ------------------------------------------------------------------ host logic with emulated kernels
def test_unet_host_logic_long_clip_vs_golden(emulated, unet_sd):
    from upscale_a_video_b200.unet_video import UNetVideoModel
    m = UNetVideoModel.from_config(_ucfg())
    m.load_state_dict(unet_sd, strict=True)
    m = m.half().eval()
    c = _unet_long_case("t12_16x24")
    sample, low, ctx = c["sample"].half(), c["low_res"].half(), c["ctx"].half()
    out = m(sample, torch.tensor(c["timestep"]), low, encoder_hidden_states=ctx, class_labels=c["class_labels"]).sample
    assert out.shape == c["out"].shape == (2, 4, 12, 16, 24) and out.dtype == torch.float16
    err = _rel(out, c["out"])
    print(f"\n[unet host-emulated t12_16x24] rel L2 err vs fp32 golden {err:.3e}")
    assert err < 5e-3


def test_propagation_host_logic_resized_flows(emulated):
    """fp32 only: the emulated recurrence step computes in fp32 and rounds once, whereas the kernel replays the reference's
    per-op fp16 rounding (a flipped consistency mask moves whole values), so fp16 is checked bit-exactly on the GPU"""
    from upscale_a_video_b200 import Propagation
    p = _load("propagation_resize.pt")
    x = p["x"]
    prop = Propagation(4, learnable=False)
    for name in ("up2x", "down2x", "ratio1_5", "t7"):
        c = p[name]
        for interp, mode, a1, a2 in PROP_MODES:
            ref = c[f"float32/{interp}_{mode}"]
            out = prop(x, c["flows_forward"], c["flows_backward"], interpolation=interp, mode=mode, fuse_scale=0.5,
                       alpha1=a1, alpha2=a2)
            assert out.shape == ref.shape and torch.equal(out, ref), (name, interp)


def test_propagation_same_shape_flows_skip_the_resize(emulated, monkeypatch):
    from upscale_a_video_b200 import Propagation
    calls = []
    monkeypatch.setattr(emu_ops, "flow_resize_area", lambda *a: calls.append(a) or flow_resize_area_standin(*a))
    x = torch.randn(1, 4, 3, 8, 12)
    prop = Propagation(4, learnable=False)
    prop(x, torch.randn(1, 2, 2, 8, 12), torch.randn(1, 2, 2, 8, 12))
    assert calls == []
    prop(x, torch.randn(1, 2, 2, 16, 24), torch.randn(1, 2, 2, 16, 24))
    assert [a[1:] for a in calls] == [((2, 8, 12), 0.5), ((2, 8, 12), 0.5)]


# ------------------------------------------------------------------ C ABI
def test_flow_resize_area_c_abi_error_convention(uav_lib):
    """null pointer or bad shape -> non-zero status + message, nothing launched (works without a GPU)"""
    from upscale_a_video_b200 import _lib
    st = uav_lib.uav_flow_resize_area(None, None, 2, 4, 32, 48, 4, 16, 24, 0.5, 0, None)
    assert st != 0 and b"null" in uav_lib.uav_last_error_string()
    buf = (C.c_uint8 * 64)()
    p = C.cast(buf, C.c_void_p)
    for bad in [(0, 4, 32, 48, 4, 16, 24), (2, 4, 32, 48, 0, 16, 24), (2, 4, 0, 48, 4, 16, 24), (2, 4, 32, 48, 4, 16, -1)]:
        st = uav_lib.uav_flow_resize_area(p, p, *bad, 0.5, 0, None)
        assert st != 0 and b"bad shape" in uav_lib.uav_last_error_string(), bad
    with pytest.raises(_lib.UavError):
        _lib.check(st, "uav_flow_resize_area")
    assert uav_lib.uav_launch_count() == 0
