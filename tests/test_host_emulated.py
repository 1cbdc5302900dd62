"""CPU check of the HOST LOGIC of the sampling path — module graph, weight packing (K-major conv filters, fused q|k|v /
k|v / temb projections, phase-collapsed upsample filters, zero-padded channels), channel-slice plumbing, prompt K/V
caching, the classifier-free-guidance shared prefix — with every kernel wrapper replaced by the plain-torch stand-ins of
`tests/emu_ops.py` (fp32 math, fp16 outputs: the kernels' contract).  Compared with the same golden vectors (minted from
the unmodified reference) and the same acceptance band as the GPU tests; the kernels themselves are covered by `-m gpu`.
The product's refusal of CPU tensors (`_lib.require_cuda`) is stubbed here and only here."""
import json
import os

import pytest
import torch

import emu_ops

G = os.path.join(os.path.dirname(__file__), "golden")
CFG = os.path.join(os.path.dirname(__file__), "..", "upscale_a_video_b200", "configs")


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.fixture()
def emulated(monkeypatch):
    from upscale_a_video_b200 import (_lib, autoencoder_kl_cond_video, layers, pipeline_upscale_a_video, propagation_module,
                                      scheduling_ddim, unet_video)
    for mod in (layers, unet_video, autoencoder_kl_cond_video, pipeline_upscale_a_video, propagation_module, scheduling_ddim):
        if hasattr(mod, "ops"):
            monkeypatch.setattr(mod, "ops", emu_ops)
    monkeypatch.setattr(_lib, "require_cuda", lambda t, who: None)


@pytest.fixture(scope="module")
def unet_sd():
    from oracle.weights import make_state_dict
    meta = json.load(open(os.path.join(G, "meta.json")))
    shapes = json.load(open(os.path.join(G, "shapes_unet.json")))
    return make_state_dict(shapes, meta["seed_unet"])


_MODELS = {}  # one instance per model for the whole module: building the 691 M-parameter UNet costs more than most tests


def _unet(unet_sd):
    if "unet" not in _MODELS:
        from upscale_a_video_b200.unet_video import UNetVideoModel
        cfg = json.load(open(os.path.join(CFG, "unet_video_config.json")))
        m = UNetVideoModel.from_config(cfg)
        m.load_state_dict(unet_sd, strict=True)
        _MODELS["unet"] = m.half().eval()
    return _MODELS["unet"]


@pytest.mark.parametrize("case", ["t3_16x24", "t2_20x28_upsize"])
def test_unet_host_logic_vs_golden(emulated, unet_sd, case):
    m = _unet(unet_sd)
    c = torch.load(os.path.join(G, "unet.pt"), weights_only=False)[case]
    sample, low, ctx = c["sample"].half(), c["low_res"].half(), c["ctx"].half()
    out = m(sample, torch.tensor(c["timestep"]), low, encoder_hidden_states=ctx, class_labels=c["class_labels"]).sample
    assert out.shape == c["out"].shape and out.dtype == torch.float16
    err = _rel(out, c["out"])
    print(f"\n[unet host-emulated {case}] rel L2 err vs fp32 golden {err:.3e}")
    assert err < 5e-3  # the GPU path measures 2.3-2.6e-3, the reference's own fp16 execution 2.8-3.2e-3
    # second call: packed weights and the prompt K/V cache are reused -> identical result
    out2 = m(sample, torch.tensor(c["timestep"]), low, encoder_hidden_states=ctx, class_labels=c["class_labels"]).sample
    assert torch.equal(out, out2)
    # a different prompt tensor must not hit the cache
    out3 = m(sample, torch.tensor(c["timestep"]), low, encoder_hidden_states=(ctx * 0.5), class_labels=c["class_labels"]).sample
    assert not torch.equal(out, out3)


def test_unet_shared_cfg_prefix_host_logic(emulated, unet_sd):
    m = _unet(unet_sd)
    c = torch.load(os.path.join(G, "unet.pt"), weights_only=False)["t3_16x24"]
    sample = c["sample"][:1].repeat(2, 1, 1, 1, 1).half()
    low = c["low_res"][:1].repeat(2, 1, 1, 1, 1).half()
    ctx = c["ctx"].half()
    a = m(sample, 601, low, encoder_hidden_states=ctx, class_labels=torch.tensor([120])).sample
    b = m(sample, 601, low, encoder_hidden_states=ctx, class_labels=torch.tensor([120]), cfg_shared_input=True).sample
    # identical math; batch-1 vs batch-2 library kernels round differently in fp32 and ~130 fp16 layers amplify that to the
    # fp16 noise floor (the GPU test measures < 2e-3 for the same comparison)
    assert _rel(b, a) < 5e-3 and not torch.equal(a[0], a[1])


def _vae(kind):
    if kind not in _MODELS:
        from oracle.weights import make_state_dict
        from upscale_a_video_b200 import AutoencoderKLVideo
        meta = json.load(open(os.path.join(G, "meta.json")))
        shapes = json.load(open(os.path.join(G, f"shapes_{kind}.json")))
        m = AutoencoderKLVideo.from_config(json.load(open(os.path.join(CFG, f"{kind}_config.json"))))
        m.load_state_dict(make_state_dict(shapes, meta["seed_vae"]), strict=True)
        _MODELS[kind] = m.eval()
    return _MODELS[kind]


def test_vae_host_logic_vs_golden(emulated):
    v = torch.load(os.path.join(G, "vae.pt"), weights_only=False)
    for kind, key in (("vae_3d", "vae3d_decode"), ("vae_video", "vaevideo_decode")):
        c = v[key]
        out = _vae(kind).decode(c["z"], c["img"], c["w_lr"]).sample
        assert out.shape == c["out"].shape and out.dtype == torch.float32
        e = _rel(out, c["out"])
        print(f"\n[{kind} decode host-emulated] rel L2 err {e:.3e}")
        assert e < 1e-2  # same band as the GPU test (measured there: 1.4-1.8e-3)
    c = v["vae3d_encode"]
    mom = _vae("vae_3d").encode(c["x"]).latent_dist.parameters
    e = _rel(mom, c["moments"])
    print(f"[vae_3d encode host-emulated] rel L2 err {e:.3e}")
    assert e < 1e-2


def test_vae_encode_odd_size_host_logic(emulated):
    """ADVICE r1: Downsample3D(padding=0) on an odd size = F.pad (0,1,0,1) + unpadded stride-2 conv -> floor((H-2)/2)+1 rows
    (resnet.py:188-192): 90 -> 45 -> 22, not 23"""
    from oracle import uav_oracle as O
    from oracle.weights import make_state_dict
    meta = json.load(open(os.path.join(G, "meta.json")))
    cfg = json.load(open(os.path.join(CFG, "vae_3d_config.json")))
    sd = make_state_dict(json.load(open(os.path.join(G, "shapes_vae_3d.json"))), meta["seed_vae"])
    g = torch.Generator().manual_seed(9)
    x = torch.rand(1, 3, 2, 90, 74, generator=g) * 2 - 1
    with torch.no_grad():
        ref = O.vae_encode_moments(sd, cfg, x)
    mom = _vae("vae_3d").encode(x).latent_dist.parameters
    assert mom.shape == ref.shape == (1, 8, 2, 22, 18)
    assert _rel(mom, ref) < 1e-2


def _hot_vae_state_dict(kind):
    """vae state dict whose up-block branch outputs are ~3e4 x larger: the decoder's residual stream leaves the fp16 range
    (what the shipped x4-upscaler VAE does: "overflows in float16", pipeline_upscale_a_video.py:667-669)"""
    from oracle.weights import make_state_dict
    meta = json.load(open(os.path.join(G, "meta.json")))
    sd = make_state_dict(json.load(open(os.path.join(G, f"shapes_{kind}.json"))), meta["seed_vae"])
    for k in sd:
        if k.startswith("decoder.up_blocks.") and (".conv2." in k or ".conv_3d." in k):
            sd[k] = sd[k] * 3.0e4
    return sd


@pytest.mark.parametrize("kind", ["vae_3d", "vae_video"])
def test_vae_decoder_residual_stream_beyond_fp16_range(emulated, monkeypatch, kind):
    """the scaled residual stream (autoencoder_kl_cond_video.VAE_STREAM_SCALE) keeps the fp16 decoder exact where an
    unscaled fp16 stream overflows"""
    from oracle import uav_oracle as O
    from upscale_a_video_b200 import AutoencoderKLVideo, autoencoder_kl_cond_video as A
    cfg = json.load(open(os.path.join(CFG, f"{kind}_config.json")))
    sd = _hot_vae_state_dict(kind)
    g = torch.Generator().manual_seed(3)
    z, img = torch.randn(1, 4, 2, 12, 16, generator=g), torch.rand(1, 3, 2, 12, 16, generator=g) * 2 - 1
    with torch.no_grad():
        taps = []
        ref = O.vae_decode(sd, cfg, z, img, 1.0)
    m = AutoencoderKLVideo.from_config(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.eval()
    out = m.decode(z, img, 1.0).sample
    e = _rel(out, ref)
    print(f"\n[{kind} hot residual stream, scale {A.VAE_STREAM_SCALE}] rel L2 err {e:.3e}")
    assert torch.isfinite(out).all() and e < 1e-2
    monkeypatch.setattr(A, "VAE_STREAM_SCALE", 1.0)
    bad = m.decode(z, img, 1.0).sample
    assert (not torch.isfinite(bad).all()) or _rel(bad, ref) > 10 * e  # the unscaled fp16 stream is what breaks


@pytest.mark.parametrize("case", ["c1_t1_64x64", "t11_16x16_prop"])
def test_pipeline_host_logic_vs_golden(emulated, unet_sd, case):
    """VideoUpscalePipeline.__call__ end to end (window plan incl. the re-anchored last window, blend, CFG, split DDIM step,
    propagation schedule, chunked decode) with emulated kernels against the reference's own pipeline output"""
    from upscale_a_video_b200 import DDIMScheduler, DDPMScheduler, Propagation, VideoUpscalePipeline
    meta = json.load(open(os.path.join(G, "meta.json")))
    c = torch.load(os.path.join(G, "pipeline.pt"), weights_only=False)[case]
    pipe = VideoUpscalePipeline(text_encoder=None, tokenizer=None, low_res_scheduler=DDPMScheduler(beta_schedule="scaled_linear"),
                                scheduler=DDIMScheduler(**meta["sched_cfgs"]["v_scaled_offset"]), vae=_vae(c["vae"]),
                                unet=_unet(unet_sd), propagator=Propagation(4, learnable=False))
    neg, pos = c["prompt_embeds"].half().chunk(2)
    out, lat = pipe(None, image=c["image"], flows_bi=c["flows"], num_inference_steps=c["steps"],
                    guidance_scale=c["guidance_scale"], noise_level=c["noise_level"], prompt_embeds=pos,
                    negative_prompt_embeds=neg, latents=c["latents"], noise=c["noise"],
                    propagation_steps=c["propagation_steps"], w_lr=c["w_lr"], return_dict=False)
    assert out.shape == c["out"].shape and out.dtype == torch.float32
    e_lat, e_img = _rel(lat, c["latents_out"]), _rel(out, c["out"])
    print(f"\n[pipeline host-emulated {case}] rel L2 err: latents {e_lat:.3e}, frames {e_img:.3e}")
    assert e_lat < 5e-2 and e_img < 5e-2  # same band as the GPU test


def test_unet_host_logic_odd_shape_vs_oracle(emulated, unet_sd):
    """a shape the fixtures do not hold: 5 frames, 18x20 (18 -> 9 -> 5 -> 3: odd sizes on the way down, explicit upsample sizes
    on the way up) against the fp32 oracle (itself pinned to the reference by the fixtures)"""
    from oracle import uav_oracle as O
    cfg = json.load(open(os.path.join(CFG, "unet_video_config.json")))
    m = _unet(unet_sd)
    g = torch.Generator().manual_seed(3)
    sample, low = torch.randn(2, 4, 5, 18, 20, generator=g), torch.randn(2, 3, 5, 18, 20, generator=g)
    ctx = torch.randn(2, 77, 1024, generator=g) * 0.3
    with torch.no_grad():
        ref = O.unet_forward(unet_sd, cfg, sample, torch.tensor(500), low, ctx, torch.tensor([120]))
    out = m(sample.half(), 500, low.half(), encoder_hidden_states=ctx.half(), class_labels=torch.tensor([120])).sample
    assert _rel(out, ref) < 5e-3


def test_pipeline_host_logic_long_clip_vs_oracle(emulated, unet_sd):
    """17 frames (windows (0,8), (6,14), re-anchored (9,17)), the conditioned video VAE, propagation at both steps, 6 decode
    chunks — against the oracle's restatement of VideoUpscalePipeline.__call__ in fp32"""
    import bench
    from oracle import uav_oracle as O
    from oracle.weights import make_state_dict
    from upscale_a_video_b200 import DDIMScheduler, DDPMScheduler, Propagation, VideoUpscalePipeline
    meta = json.load(open(os.path.join(G, "meta.json")))
    scfg = meta["sched_cfgs"]["v_scaled_offset"]
    T, H, W, steps, prop = 17, 8, 8, 2, [0, 1]
    image, fw, bw, pe = bench.synth_inputs(T, H, W, "cpu")
    g = torch.Generator().manual_seed(5)
    noise, lat0 = torch.randn(1, 3, T, H, W, generator=g), torch.randn(1, 4, T, H, W, generator=g)
    pipe = VideoUpscalePipeline(None, None, DDPMScheduler(beta_schedule="scaled_linear"), DDIMScheduler(**scfg), _vae("vae_video"),
                                _unet(unet_sd), Propagation(4, learnable=False))
    neg, pos = pe.half().chunk(2)
    out, lat = pipe(None, image=image, flows_bi=[fw, bw], num_inference_steps=steps, guidance_scale=6.0, noise_level=120,
                    prompt_embeds=pos, negative_prompt_embeds=neg, latents=lat0, noise=noise, propagation_steps=prop,
                    return_dict=False)
    ucfg = json.load(open(os.path.join(CFG, "unet_video_config.json")))
    vcfg = json.load(open(os.path.join(CFG, "vae_video_config.json")))
    vsd = make_state_dict(json.load(open(os.path.join(G, "shapes_vae_video.json"))), meta["seed_vae"])
    with torch.no_grad():
        ref, ref_lat = O.pipeline_call(unet_sd, ucfg, vsd, vcfg, O.DDIM(**scfg), O.DDIM(beta_schedule="scaled_linear"), image=image,
                                       prompt_embeds=pe, noise=noise, latents=lat0, flows_bi=[fw, bw], num_inference_steps=steps,
                                       guidance_scale=6.0, noise_level=120, propagation_steps=prop, return_latents=True)
    assert _rel(lat, ref_lat) < 5e-2 and _rel(out, ref) < 5e-2


SHARD_WORKER = r"""
import json, os, sys
root = sys.argv[1]
sys.path[:0] = [root, os.path.join(root, "tests")]
import torch, torch.distributed as dist
import bench, emu_ops
from oracle.weights import make_state_dict
from upscale_a_video_b200 import (_lib, autoencoder_kl_cond_video, layers, pipeline_upscale_a_video, propagation_module,
                                  scheduling_ddim, unet_video)
for mod in (layers, unet_video, autoencoder_kl_cond_video, pipeline_upscale_a_video, propagation_module, scheduling_ddim):
    if hasattr(mod, "ops"):
        mod.ops = emu_ops
_lib.require_cuda = lambda t, who: None
from upscale_a_video_b200 import AutoencoderKLVideo, DDIMScheduler, DDPMScheduler, Propagation, UNetVideoModel, VideoUpscalePipeline
torch.set_num_threads(4)
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
solo = [dist.new_group([r]) for r in range(world)][rank]
G, CFG = os.path.join(root, "tests", "golden"), os.path.join(root, "upscale_a_video_b200", "configs")
meta = json.load(open(os.path.join(G, "meta.json")))
unet = UNetVideoModel.from_config(json.load(open(os.path.join(CFG, "unet_video_config.json"))))
unet.load_state_dict(make_state_dict(json.load(open(os.path.join(G, "shapes_unet.json"))), meta["seed_unet"]), strict=True)
vae = AutoencoderKLVideo.from_config(json.load(open(os.path.join(CFG, "vae_3d_config.json"))))
vae.load_state_dict(make_state_dict(json.load(open(os.path.join(G, "shapes_vae_3d.json"))), meta["seed_vae"]), strict=True)
pipe = VideoUpscalePipeline(None, None, DDPMScheduler(beta_schedule="scaled_linear"),
                            DDIMScheduler(**meta["sched_cfgs"]["v_scaled_offset"]), vae.eval(), unet.half().eval(),
                            Propagation(4, learnable=False))
T, H, W = 14, 8, 8  # two unique windows per step, five decode chunks (3 + 2 per rank, ragged last chunk)
image, fw, bw, pe = bench.synth_inputs(T, H, W, "cpu")
g = torch.Generator().manual_seed(5)
noise, lat0 = torch.randn(1, 3, T, H, W, generator=g), torch.randn(1, 4, T, H, W, generator=g)
neg, pos = pe.half().chunk(2)
kw = dict(image=image, flows_bi=[fw, bw], num_inference_steps=1, guidance_scale=6.0, noise_level=120, prompt_embeds=pos,
          negative_prompt_embeds=neg, latents=lat0, noise=noise, propagation_steps=[0], return_dict=False)
calls = {"n": 0}
orig_forward = unet.forward
def counting(*a, **k):
    calls["n"] += 1
    return orig_forward(*a, **k)
unet.forward = counting
pipe.process_group = solo
out1, lat1 = pipe(None, **kw)
n_solo = calls["n"]
calls["n"] = 0
pipe.process_group = None
out2, lat2 = pipe(None, **kw)
assert n_solo == 2 and calls["n"] == 1, (n_solo, calls["n"])  # 2 windows alone, 1 window per rank when sharded
assert torch.equal(lat1, lat2) and torch.equal(out1, out2), ((lat1 - lat2).abs().max(), (out1 - out2).abs().max())
# 20 frames = 3 unique windows on 2 ranks: dealt as 6 CFG-half units (3 single-half calls per rank instead of 2 rounds of whole
# windows).  The dealing / gather / blend-order logic does not depend on what the UNet computes, so this part runs a tiny
# stand-in UNet and decoder (per-batch-item deterministic functions): sharded == unsharded bit for bit.
from upscale_a_video_b200 import sharding
assert sharding.window_units(3, 2, True) == [(0, 0), (0, 1), (1, 0), (1, 1), (2, 0), (2, 1)]
from types import SimpleNamespace
class TinyUNet:
    config = SimpleNamespace(in_channels=7)
    calls = 0
    def forward(self, sample, timestep, low_res, encoder_hidden_states=None, class_labels=None, cfg_shared_input=False):
        TinyUNet.calls += 1
        m = encoder_hidden_states.float().mean(dim=(1, 2)).view(-1, 1, 1, 1, 1)
        y = torch.tanh(sample.float() * 0.7 + low_res.float().mean(1, keepdim=True) * 0.3 + m + 0.001 * float(timestep))
        return SimpleNamespace(sample=y.to(sample.dtype))
    __call__ = forward
class TinyVAE:
    config = SimpleNamespace(latent_channels=4, out_channels=3, scaling_factor=0.08333)
    def decode(self, z, img=None, w_lr=1, latent_scale=1.0, clamp=False):
        up = (z.float() * latent_scale)[:, :3].repeat_interleave(4, dim=-2).repeat_interleave(4, dim=-1)
        return SimpleNamespace(sample=up.clamp(-1, 1) if clamp else up)
tiny = VideoUpscalePipeline(None, None, DDPMScheduler(beta_schedule="scaled_linear"),
                            DDIMScheduler(**meta["sched_cfgs"]["v_scaled_offset"]), TinyVAE(), TinyUNet(), Propagation(4, learnable=False))
T = 20
image, fw, bw, pe = bench.synth_inputs(T, H, W, "cpu")
noise, lat0 = torch.randn(1, 3, T, H, W, generator=g), torch.randn(1, 4, T, H, W, generator=g)
kw.update(image=image, flows_bi=[fw, bw], latents=lat0, noise=noise, num_inference_steps=2, propagation_steps=[1])
tiny.process_group = solo
out1, lat1 = tiny(None, **kw)
n_solo, TinyUNet.calls = TinyUNet.calls, 0
tiny.process_group = None
out2, lat2 = tiny(None, **kw)
assert n_solo == 6 and TinyUNet.calls == 6, (n_solo, TinyUNet.calls)  # 3 windows x 2 steps alone; 3 half-calls x 2 steps per rank
assert torch.equal(lat1, lat2) and torch.equal(out1, out2)
dist.barrier()
if rank == 0:
    print("SHARDED_PIPELINE_OK")
"""


def test_sharded_pipeline_gloo_world2(tmp_path):
    """the whole N > 1 data path on CPU: two ranks (gloo) run VideoUpscalePipeline.__call__ with emulated kernels; windows of a
    DDIM step and decode chunks are dealt to ranks, gathered once per step / once at the end, and every rank ends with a
    result bit-identical to its own unsharded run (half the UNet calls)"""
    import subprocess
    import sys
    script = tmp_path / "shard_worker.py"
    script.write_text(SHARD_WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29523", str(script), root], capture_output=True, text=True, env=env,
                       timeout=1500)
    assert r.returncode == 0 and "SHARDED_PIPELINE_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_color_correction_host_logic_vs_reference_fixtures(monkeypatch):
    """color_correction.py (AdaIN, wavelet chains with their ping-pong buffers, the CLI block, packing) with emulated kernels
    against the fixtures minted from the reference's own functions"""
    from upscale_a_video_b200 import _lib, color_correction as cc
    monkeypatch.setattr(cc, "ops", emu_ops)
    monkeypatch.setattr(_lib, "require_cuda", lambda t, who: None)
    cases = torch.load(os.path.join(G, "color.pt"), map_location="cpu", weights_only=False)
    for name, c in cases.items():
        lr, hr, up = c["lr"], c["hr"], c["bicubic"]
        assert (cc.upsample_lr_frames(lr, 4) - up).abs().max().item() < 2e-6
        assert (cc.adaptive_instance_normalization(hr, up) - c["adain"]).abs().max().item() < 5e-6, name
        assert (cc.wavelet_reconstruction(hr, up) - c["wavelet"]).abs().max().item() < 2e-6, name
        if "high" in c:
            high, low = cc.wavelet_decomposition(hr)
            assert (high - c["high"]).abs().max().item() < 2e-6 and (low - c["low"]).abs().max().item() < 1e-6
        out = cc.color_fix_frames(hr.permute(1, 0, 2, 3)[None], lr.permute(1, 0, 2, 3)[None], "AdaIn")
        assert (out - c["adain"]).abs().max().item() < 1e-5
        assert torch.equal(cc.pack_video_uint8(hr), c["pack_hr"])
    with pytest.raises(ValueError):
        cc.color_fix_frames(hr.permute(1, 0, 2, 3)[None], lr.permute(1, 0, 2, 3)[None], "bogus")
