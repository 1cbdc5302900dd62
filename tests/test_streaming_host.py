"""CPU checks of the streaming output path: `VideoUpscalePipeline.sample_latents` + `decode_chunks`, the streaming tile
driver `tiling.iter_upscale_tiled`, and the command's chunk-by-chunk writing loop, alone and over two gloo ranks.  Kernels
are the plain-torch stand-ins of `tests/emu_ops.py`; where only the data flow matters, tiny stand-in models keep it fast."""
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import emu_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
CFG = os.path.join(ROOT, "upscale_a_video_b200", "configs")


def emulate():
    """every kernel wrapper of the sampling path and the colour fix -> emu_ops; returns the undo list"""
    from upscale_a_video_b200 import (_lib, autoencoder_kl_cond_video, color_correction, layers, pipeline_upscale_a_video,
                                      propagation_module, scheduling_ddim, unet_video)
    undo = [(_lib, "require_cuda", _lib.require_cuda)]
    _lib.require_cuda = lambda t, who: None
    for mod in (layers, unet_video, autoencoder_kl_cond_video, pipeline_upscale_a_video, propagation_module,
                scheduling_ddim, color_correction):
        undo.append((mod, "ops", mod.ops))
        mod.ops = emu_ops
    return undo


@pytest.fixture()
def emulated():
    undo = emulate()
    yield
    for mod, name, v in undo:
        setattr(mod, name, v)


class TinyUNet:
    """per-batch-item deterministic stand-in of UNetVideoModel"""
    config = SimpleNamespace(in_channels=7)

    def forward(self, sample, timestep, low_res, encoder_hidden_states=None, class_labels=None, cfg_shared_input=False):
        m = encoder_hidden_states.float().mean(dim=(1, 2)).view(-1, 1, 1, 1, 1)
        y = torch.tanh(sample.float() * 0.7 + low_res.float().mean(1, keepdim=True) * 0.3 + m + 0.001 * float(timestep))
        return SimpleNamespace(sample=y.to(sample.dtype))

    __call__ = forward


class TinyVAE:
    """frame-wise stand-in of the conditioned decoder; records the frame count of every decode"""
    config = SimpleNamespace(latent_channels=4, out_channels=3, scaling_factor=0.08333)

    def __init__(self):
        self.frames = []

    def decode(self, z, img=None, w_lr=1, latent_scale=1.0, clamp=False):
        self.frames.append(z.shape[2])
        up = (z.float() * latent_scale)[:, :3] + w_lr * img.float()
        up = up.repeat_interleave(4, dim=-2).repeat_interleave(4, dim=-1)
        return SimpleNamespace(sample=up.clamp(-1, 1) if clamp else up)


def make_pipeline(unet, vae):
    from upscale_a_video_b200 import DDIMScheduler, DDPMScheduler, Propagation, VideoUpscalePipeline
    meta = json.load(open(os.path.join(G, "meta.json")))
    return VideoUpscalePipeline(None, None, DDPMScheduler(beta_schedule="scaled_linear"),
                                DDIMScheduler(**meta["sched_cfgs"]["v_scaled_offset"]), vae, unet,
                                Propagation(4, learnable=False))


def pipeline_kwargs(T, H=8, W=8, steps=2):
    """14 frames: two unique UNet windows per step, five decode chunks, the last one 2 frames"""
    import bench
    image, fw, bw, pe = bench.synth_inputs(T, H, W, "cpu")
    g = torch.Generator().manual_seed(5)
    noise, lat0 = torch.randn(1, 3, T, H, W, generator=g), torch.randn(1, 4, T, H, W, generator=g)
    neg, pos = pe.half().chunk(2)
    return dict(image=image, flows_bi=[fw, bw], num_inference_steps=steps, guidance_scale=6.0, noise_level=120,
                prompt_embeds=pos, negative_prompt_embeds=neg, latents=lat0, noise=noise, propagation_steps=[0, 1],
                w_lr=0.5)


def test_sample_then_decode_chunks_equals_call(emulated):
    """`__call__` == `sample_latents` + concatenated `decode_chunks`, bit for bit, with the conditioned vae_video decoder
    and propagation; 14 frames decode as 3 + 3 + 3 + 3 + 2"""
    from oracle.weights import make_state_dict
    from upscale_a_video_b200 import AutoencoderKLVideo
    meta = json.load(open(os.path.join(G, "meta.json")))
    vae = AutoencoderKLVideo.from_config(json.load(open(os.path.join(CFG, "vae_video_config.json"))))
    vae.load_state_dict(make_state_dict(json.load(open(os.path.join(G, "shapes_vae_video.json"))), meta["seed_vae"]),
                        strict=True)
    assert vae.decoder.condition_img
    pipe = make_pipeline(TinyUNet(), vae.eval())
    kw = pipeline_kwargs(14)
    images, lat = pipe(None, **kw, return_dict=False)
    sampled = pipe.sample_latents(None, **kw)
    chunks = list(pipe.decode_chunks(sampled))
    assert [(s, e) for s, e, _ in chunks] == [(0, 3), (3, 6), (6, 9), (9, 12), (12, 14)]
    for s, e, f in chunks:
        assert f.shape == (1, 3, e - s, 32, 32) and f.dtype == torch.float32
    assert sampled.latents.dtype == torch.float32 and sampled.image_dec.dtype == torch.float32 and sampled.w_lr == 0.5
    assert torch.equal(torch.cat([f for _, _, f in chunks], dim=2), images)
    assert torch.equal(sampled.latents, lat)
    assert images.abs().max() <= 1.0 and images.std() > 0.05  # clamped and not degenerate


# -------------------------------------------------------------------------------- tile driver stand-ins
class _TileStub:
    def __init__(self):
        self.process_group = None
        self.vae = SimpleNamespace(config=SimpleNamespace(latent_channels=4, out_channels=3))
        self.text_encoder = SimpleNamespace(dtype=torch.float32)
        self.decoded = []  # frame count of every decode

    def _sample(self, prompt=None, image=None, flows_bi=None, generator=None, noise=None, latents=None, w_lr=1, **kw):
        import torch.distributed as dist
        from upscale_a_video_b200.pipeline_upscale_a_video import randn_tensor
        assert self.process_group is None or dist.get_world_size(self.process_group) == 1  # no nested sharding
        if noise is None:
            noise = randn_tensor(image.shape, generator=generator, dtype=torch.float32)
        if latents is None:
            latents = randn_tensor((image.shape[0], 4, *image.shape[2:]), generator=generator, dtype=torch.float32)
        lat = latents.float() * 0.25 + noise.float().mean(1, keepdim=True) * 0.1
        if flows_bi is not None:
            lat[:, :, 1:] += 0.01 * flows_bi[0].float().mean(1, keepdim=True)
        return SimpleNamespace(latents=lat, image_dec=image.clone().float(), w_lr=w_lr)

    def decode_latents_vsr(self, latents, img, w_lr):
        self.decoded.append(latents.shape[2])
        up = torch.tanh(latents[:, :3] + w_lr * img + 0.5 * latents[:, 3:])  # frame by frame, as the VAE decodes
        return up.repeat_interleave(4, dim=-2).repeat_interleave(4, dim=-1)


class StreamingStub(_TileStub):
    """what iter_upscale_tiled and the command use: sample_latents / decode_latents_vsr / decode_chunks"""
    sample_latents = _TileStub._sample

    @property
    def decode_chunks(self):
        from upscale_a_video_b200 import VideoUpscalePipeline
        return VideoUpscalePipeline.decode_chunks.__get__(self)


class CallOnlyStub(_TileStub):
    """the same model behind `__call__` alone: the whole clip in one decode"""
    def __call__(self, **kw):
        r = self._sample(**kw)
        return SimpleNamespace(images=self.decode_latents_vsr(r.latents, r.image_dec, r.w_lr))


def tiled_case():
    """(image, flows) of 14 frames on a 2 x 3 tile plan (tile 32, overlap 16: the tiles overlap and the last row is
    merged)"""
    t, h, w = 14, 70, 90
    g = torch.Generator().manual_seed(3)
    image = torch.rand(1, 3, t, h, w, generator=g) * 2 - 1
    flows = [torch.randn(1, 2, t - 1, h, w, generator=g), torch.randn(1, 2, t - 1, h, w, generator=g)]
    return image, flows


def check_tiled_streaming(process_group=None):
    from upscale_a_video_b200 import sharding, tiling
    image, flows = tiled_case()
    plan = tiling.plan_tiles(image.shape[-2], image.shape[-1], 32, 16)
    assert len(plan) == 6
    whole_pipe, stream_pipe = CallOnlyStub(), StreamingStub()
    whole = tiling.upscale_tiled(whole_pipe, image, flows, torch.Generator().manual_seed(10), tile_size=32, overlap=16,
                                 process_group=process_group, w_lr=0.7)
    got = list(tiling.iter_upscale_tiled(stream_pipe, image, flows, torch.Generator().manual_seed(10), tile_size=32,
                                         overlap=16, process_group=process_group, w_lr=0.7))
    assert [(s, e) for s, e, _ in got] == sharding.decode_chunks(14)
    assert torch.equal(torch.cat([c for _, _, c in got], dim=2), whole)
    rank, world = sharding.world_info(process_group)
    mine = len([i for i in range(len(plan)) if i % world == rank])
    assert whole_pipe.decoded == [14] * mine
    assert max(stream_pipe.decoded) <= 3 and sum(stream_pipe.decoded) == 14 * mine
    assert stream_pipe.process_group is None
    return whole


def test_iter_upscale_tiled_equals_upscale_tiled():
    whole = check_tiled_streaming()
    assert whole.std() > 0.1


# -------------------------------------------------------------------------------- the command loop
def patch_command(monkeypatch_setattr, pipe, recorder):
    """cli.main on CPU: no checkpoints, no GPU; `recorder` collects every mp4 / PNG write"""
    from upscale_a_video_b200 import cli, color_correction, video_io

    def pack_video(frames):
        return emu_ops.pack_video_uint8(frames)

    def pack_png(frames):
        return ((frames.float() + 1) / 2 * 255 + 0.5).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()

    real_write, real_frames = video_io.VideoWriter.write, video_io.write_frames

    def write(self, frames_rgb):
        recorder.append(("mp4", os.path.basename(self.path), len(frames_rgb)))
        real_write(self, frames_rgb)

    def write_frames(folder, frames_rgb, start=0):
        recorder.append(("png", start, len(frames_rgb)))
        return real_frames(folder, frames_rgb, start=start)

    def ingest(frames, device, from_video):
        x = torch.from_numpy(frames[..., ::-1].copy()).permute(3, 0, 1, 2)[None].float()
        return x / 127.5 - 1

    for obj, name, value in ((cli, "checkpoint_paths", lambda args: {}),
                             (cli, "_init_distributed", lambda: (torch.device("cpu"), False)),
                             (cli, "load_models", lambda args, paths, device: (pipe, None)),
                             (cli, "ingest_frames", ingest),
                             (torch.cuda, "synchronize", lambda device=None: None),
                             (color_correction, "pack_video_uint8", pack_video),
                             (color_correction, "pack_frames_png", pack_png),
                             (video_io.VideoWriter, "write", write),
                             (video_io, "write_frames", write_frames)):
        monkeypatch_setattr(obj, name, value)


def write_clip(folder, t, h, w):
    from upscale_a_video_b200 import video_io
    rgb = np.random.default_rng(t + h + w).integers(0, 256, size=(t, h, w, 3), dtype=np.uint8)
    video_io.write_frames(str(folder), rgb)


def check_command_outputs(out, name, t, recorder):
    from upscale_a_video_b200 import video_io
    mp4 = [r for r in recorder if r[0] == "mp4"]
    assert [r[2] for r in mp4] == [3] * (t // 3) + ([t % 3] if t % 3 else [])  # in order, at most 3 frames each
    pngs = [r for r in recorder if r[0] == "png"]
    assert [r[1] for r in pngs] == list(range(0, t, 3)) and sum(r[2] for r in pngs) == t
    assert sorted(os.listdir(out / "frame" / name)) == [f"{i:04d}.png" for i in range(t)]
    frames, _, _ = video_io.read_frames(str(out / "video" / f"{name}.mp4"))
    assert frames.shape[0] == t
    return video_io.read_frames(str(out / "frame" / name))[0]


@pytest.mark.parametrize("tiled", [False, True])
def test_command_streams_chunks_to_disk(tmp_path, monkeypatch, emulated, tiled):
    """each write gets at most 3 frames in time order, PNG numbering runs without gaps, the mp4 has every frame, and
    the frames equal the whole-clip path (pipeline output -> colour fix -> PNG rounding)"""
    pytest.importorskip("cv2")
    from upscale_a_video_b200 import cli, color_correction, tiling
    t, h, w = 14, 12, 80
    write_clip(tmp_path / "clip", t, h, w)
    pipe, recorder = StreamingStub(), []
    patch_command(monkeypatch.setattr, pipe, recorder)
    extra = ["--perform_tile", "--tile_size", "8"] if tiled else []
    out = tmp_path / "out"
    written = cli.main(["-i", str(tmp_path / "clip"), "-o", str(out), "--color_fix", "AdaIn", "--save_image", *extra])
    name = "clip_n120_g6_s30"
    assert written == [str(out / "video" / f"{name}.mp4")]
    got = check_command_outputs(out, name, t, recorder)
    assert max(pipe.decoded) <= 3
    # the whole-clip library path on the same stand-ins
    from upscale_a_video_b200 import video_io
    bgr, _, _ = video_io.read_frames(str(tmp_path / "clip"))
    vframes = cli.ingest_frames(bgr, "cpu", False)
    g = torch.Generator().manual_seed(cli.SEED)
    kw = dict(num_inference_steps=30, guidance_scale=6, noise_level=120, negative_prompt="blur, worst quality",
              propagation_steps=[], prompt="best quality, extremely detailed")
    if tiled:
        whole = tiling.upscale_tiled(CallOnlyStub(), vframes, None, g, tile_size=8, overlap=64, **kw)
    else:
        whole = CallOnlyStub()(image=vframes, generator=g, **kw).images
    ref = color_correction.pack_frames_png(color_correction.color_fix_frames(whole, vframes, "AdaIn")).numpy()
    assert np.array_equal(got[..., ::-1], ref)


def test_command_failure_mid_clip_leaves_no_mp4(tmp_path, monkeypatch, emulated):
    pytest.importorskip("cv2")
    from upscale_a_video_b200 import cli
    write_clip(tmp_path / "clip", 14, 12, 80)
    pipe, recorder = StreamingStub(), []
    patch_command(monkeypatch.setattr, pipe, recorder)
    real = pipe.decode_latents_vsr

    def failing(latents, img, w_lr):
        if len(pipe.decoded) == 2:
            raise RuntimeError("decode failed")
        return real(latents, img, w_lr)

    pipe.decode_latents_vsr = failing
    out = tmp_path / "out"
    with pytest.raises(RuntimeError, match="decode failed"):
        cli.main(["-i", str(tmp_path / "clip"), "-o", str(out), "--save_image"])
    assert [r[0] for r in recorder] == ["png", "mp4", "png", "mp4"]  # two chunks went out before the failure
    assert os.listdir(out / "video") == []


# -------------------------------------------------------------------------------- two gloo ranks
WORKER = r"""
import os, sys
root = sys.argv[1]
sys.path[:0] = [root, os.path.join(root, "tests")]
import torch, torch.distributed as dist
torch.set_num_threads(2)
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
import test_streaming_host as H
from upscale_a_video_b200 import sharding
H.emulate()
solo = [dist.new_group([r]) for r in range(world)][rank]

# 1. decode_chunks: every rank yields all 5 chunks of 14 frames, equal to its own unsharded run; chunk k decoded by
#    rank k % 2; 3 grouped gathers, the last one ragged (one chunk for two ranks)
vae = H.TinyVAE()
pipe = H.make_pipeline(H.TinyUNet(), vae)
kw = H.pipeline_kwargs(14)
pipe.process_group = solo
alone = [c for c in pipe.decode_chunks(pipe.sample_latents(None, **kw))]
pipe.process_group = None
sampled = pipe.sample_latents(None, **kw)
vae.frames.clear()
gathers = []
real_gather = sharding.all_gather_units
def counting(local, n_units, *a, **k):
    gathers.append(n_units)
    return real_gather(local, n_units, *a, **k)
sharding.all_gather_units = counting
shared = list(pipe.decode_chunks(sampled))
sharding.all_gather_units = real_gather
assert gathers == [2, 2, 1], gathers
assert vae.frames == ([3, 3, 2] if rank == 0 else [3, 3]), vae.frames
assert [(s, e) for s, e, _ in shared] == [(0, 3), (3, 6), (6, 9), (9, 12), (12, 14)]
for (s, e, a), (_, _, b) in zip(alone, shared):
    assert a.shape == b.shape == (1, 3, e - s, 32, 32) and torch.equal(a, b), (s, e)

# 2. iter_upscale_tiled == upscale_tiled over two ranks
H.check_tiled_streaming()

# 3. the command over two ranks: rank 0 alone writes, the frames equal the single-process run
from pathlib import Path
from upscale_a_video_b200 import cli
class Setter:
    def __call__(self, obj, name, value):
        setattr(obj, name, value)
tmp = Path(sys.argv[2])
for tiled in (False, True):
    stub, recorder = H.StreamingStub(), []
    H.patch_command(Setter(), stub, recorder)
    extra = ["--perform_tile", "--tile_size", "8"] if tiled else []
    out = tmp / f"two_{tiled}"
    written = cli.main(["-i", str(tmp / "clip"), "-o", str(out), "--save_image", *extra])
    name = "clip_n120_g6_s30"
    if rank == 0:
        assert written == [str(out / "video" / f"{name}.mp4")]
        got = H.check_command_outputs(out, name, 14, recorder)
        one = tmp / f"one_{tiled}" / "frame" / name
        from upscale_a_video_b200 import video_io
        assert (got == video_io.read_frames(str(one))[0]).all()
    else:
        assert written == [] and recorder == [], recorder
    assert max(stub.decoded) <= 3
    dist.barrier()
dist.barrier()
if rank == 0:
    print("STREAMING_WORLD2_OK")
"""


def test_streaming_gloo_world2(tmp_path, monkeypatch):
    """two gloo ranks: grouped chunk gathers (ragged last group), the streaming tile driver and the command loop give
    every rank the single-process result, and only rank 0 writes"""
    pytest.importorskip("cv2")
    from upscale_a_video_b200 import cli
    write_clip(tmp_path / "clip", 14, 12, 80)
    for tiled in (False, True):  # the single-process runs the ranks compare against
        stub, recorder = StreamingStub(), []
        with monkeypatch.context() as m:
            patch_command(m.setattr, stub, recorder)
            extra = ["--perform_tile", "--tile_size", "8"] if tiled else []
            cli.main(["-i", str(tmp_path / "clip"), "-o", str(tmp_path / f"one_{tiled}"), "--save_image", *extra])
    script = tmp_path / "streaming_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29537", str(script), ROOT, str(tmp_path)], capture_output=True,
                       text=True, env=env, timeout=900)
    assert r.returncode == 0 and "STREAMING_WORLD2_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
