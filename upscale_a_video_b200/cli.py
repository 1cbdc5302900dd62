"""`python -m upscale_a_video_b200`: upscale video files x4 end to end.

The reference's `inference_upscale_a_video.py` with its flags, defaults and output layout, on the uav_b200 pipeline:

    python -m upscale_a_video_b200 -i inputs/clip.mp4 -o results -p 24,26,28 --color_fix Wavelet

Per clip: uint8 frames are copied to the GPU and normalised (and area-downsampled by 4 when both sides are >= 1280) by
`ops.unpack_video_uint8`; RAFT flows when `-p` is given; the pipeline's sampling, whole or per tile
(`tiling.iter_upscale_tiled`); then, 3 frames at a time, the decode, the colour fix, uint8 packing on the GPU for the
mp4 (`pack_video_uint8`) and, with `--save_image`, for the PNG frames (`pack_frames_png`, save_image's rounding), and the
writes.  No buffer at output resolution holds more than one 3-frame chunk, so memory does not grow with clip length
beyond the low-resolution sampling state.  Under `torchrun` (WORLD_SIZE > 1) each process drives the GPU LOCAL_RANK
and the pipeline's tile / window sharding splits the work; only rank 0 writes files.

With `--llava_path` (and without `--no_llava`) frame 0 of each clip is captioned by `llava.LLavaAgent` before the
upscale, with the reference's preprocessing and a generator seeded from SEED; the prompt is `caption + a_prompt`.  When
clip i is reached and has no caption yet, the first frames of clips i .. i + CAPTION_BATCH - 1 are captioned in one
call, each with its own generator seeded SEED, which gives each clip the caption a call on it alone gives.  Under
`torchrun` only rank 0 loads and runs the captioner and the captions are broadcast to the other ranks.
`--llava_int8` loads the captioner with weight-only int8 decoder and projector Linears (`weights="int8"`).

Deliberate differences from the reference CLI (INTEGRATION.md §3): the captioner runs only when `--llava_path` names a
LLaVA-1.5 folder (otherwise `--caption` supplies the caption text), its sampling is seeded, errors raise instead of
being printed, `--save_image` writes one PNG per frame, the mp4 codec is
mp4v, and the tiling decision is taken per clip."""
from __future__ import annotations

import argparse
import contextlib
import os
import textwrap
import time
from typing import Iterator, List, Optional, Tuple

import numpy as np
import torch

from . import color_correction, ops, tiling, video_io

TILE_OVERLAP = 64  # inference_upscale_a_video.py:210
SEED = 10          # inference_upscale_a_video.py:197


def str_to_list(value: str) -> List[int]:
    return list(map(int, value.split(",")))


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="python -m upscale_a_video_b200",
                                description="Upscale videos x4 with Upscale-A-Video on the GPU.")
    p.add_argument("-i", "--input_path", type=str, default="./inputs",
                   help="A video file, a folder of frames, or a folder of videos.")
    p.add_argument("-o", "--output_path", type=str, default="./results", help="Output folder.")
    p.add_argument("-n", "--noise_level", type=int, default=120,
                   help="Noise level [0, 200] applied to the input video. Default: 120")
    p.add_argument("-g", "--guidance_scale", type=int, default=6,
                   help="Classifier-free guidance scale for prompts. Default: 6")
    p.add_argument("-s", "--inference_steps", type=int, default=30, help="Number of denoising steps. Default: 30")
    p.add_argument("-p", "--propagation_steps", type=str_to_list, default=[],
                   help="Comma-separated denoising steps after which latents are propagated along RAFT flows.")
    p.add_argument("--a_prompt", type=str, default="best quality, extremely detailed")
    p.add_argument("--n_prompt", type=str, default="blur, worst quality")
    p.add_argument("--use_video_vae", action="store_true", default=False)
    p.add_argument("--color_fix", type=str, default="None", choices=["None", "AdaIn", "Wavelet"])
    p.add_argument("--no_llava", action="store_true", default=False, help="Do not caption, even with --llava_path.")
    p.add_argument("--load_8bit_llava", action="store_true", default=False,
                   help="Not supported (bitsandbytes' LLM.int8()); see --llava_int8.")
    p.add_argument("--llava_path", type=str, default=None,
                   help="LLaVA-1.5 folder (released format): caption frame 0 of each clip with it.")
    p.add_argument("--llava_vision_path", type=str, default=None,
                   help="CLIP ViT-L/14-336 folder of the captioner's vision tower (default: the config's mm_vision_tower).")
    p.add_argument("--llava_int8", action="store_true", default=False,
                   help="Hold the captioner's decoder and projector Linears as weight-only int8 (about half the memory "
                        "of fp16, and half the bytes per decoded token).")
    p.add_argument("--perform_tile", action="store_true", default=False)
    p.add_argument("--tile_size", type=int, default=256)
    p.add_argument("--save_image", action="store_true", default=False)
    p.add_argument("--save_suffix", type=str, default="")
    p.add_argument("--model_dir", type=str, default="./pretrained_models/upscale_a_video",
                   help="Folder of the released checkpoints (text_encoder/, tokenizer/, vae/, unet/, ...).")
    p.add_argument("--caption", type=str, default="",
                   help="Caption text prepended to --a_prompt (stands in for the LLaVA caption).")
    return p


def parse_args(argv: Optional[List[str]] = None) -> argparse.Namespace:
    parser = build_parser()
    args = parser.parse_args(argv)
    if args.load_8bit_llava:
        parser.error("--load_8bit_llava: there is no LLaVA captioner for bitsandbytes' LLM.int8() (int8 activations); "
                     "--llava_int8 runs it on weight-only int8 Linears")
    if args.llava_int8 and not use_llava(args):
        parser.error("--llava_int8 needs the captioner: pass --llava_path (without --no_llava)")
    if args.caption and use_llava(args):
        parser.error("--caption and --llava_path both give the caption: pass one of them (or --no_llava)")
    return args


def use_llava(args: argparse.Namespace) -> bool:
    return args.llava_path is not None and not args.no_llava


def caption_frame(agent, frame_bgr: np.ndarray) -> str:
    """inference_upscale_a_video.py:158-175: the caption of a clip's first frame, sampled from a generator seeded with
    SEED so that a rerun gives the same caption"""
    from .llava import frame0_image
    img = frame0_image(np.ascontiguousarray(frame_bgr[..., ::-1]))
    return agent.gen_image_caption([img], generator=torch.Generator().manual_seed(SEED))[0]


def caption_frames(agent, frames_bgr: List[np.ndarray]) -> List[str]:
    """`caption_frame` of each frame, from one `gen_image_caption` call with one generator seeded SEED per frame"""
    from .llava import frame0_image
    imgs = [frame0_image(np.ascontiguousarray(f[..., ::-1])) for f in frames_bgr]
    return agent.gen_image_caption(imgs, generator=[torch.Generator().manual_seed(SEED) for _ in imgs])


def _shared_captions(agent, first_frame, video_paths: List[str], rank: int) -> List[str]:
    """the captions of the clips `video_paths`, whose first clip's frame 0 is `first_frame`: rank 0 reads the other
    clips' first frames and captions them all in one call; under torch.distributed every rank gets the list"""
    import torch.distributed as dist
    captions = None
    if rank == 0:
        frames = [first_frame] + [video_io.read_first_frame(p) for p in video_paths[1:]]
        captions = caption_frames(agent, frames)
    if dist.is_initialized() and dist.get_world_size() > 1:
        box = [captions]
        dist.broadcast_object_list(box, src=0)
        captions = box[0]
    return captions


def save_name(video_name: str, args: argparse.Namespace) -> str:
    """inference_upscale_a_video.py:341-343"""
    prop = "_p" + "_".join(map(str, args.propagation_steps)) if args.propagation_steps else ""
    suffix = "_" + args.save_suffix if args.save_suffix else ""
    return f"{video_name}_n{args.noise_level}_g{args.guidance_scale}_s{args.inference_steps}{prop}{suffix}"


def output_paths(args: argparse.Namespace, video_name: str):
    """(mp4 path, PNG folder) of one clip"""
    name = save_name(video_name, args)
    return os.path.join(args.output_path, "video", f"{name}.mp4"), os.path.join(args.output_path, "frame", name)


def lr_size(h: int, w: int):
    """inference_upscale_a_video.py:183-185: frames of at least 1280 x 1280 are area-downsampled by 4 before sampling"""
    return (h // 4, w // 4) if h >= 1280 and w >= 1280 else (h, w)


def ingest_frames(frames_bgr: np.ndarray, device, from_video: bool) -> torch.Tensor:
    """(t, h, w, 3) uint8 BGR host frames -> (1, 3, t, h', w') fp32 RGB in [-1, 1] on `device` (inference…:180-188).
    One byte per sample crosses the bus; normalisation and resize run in one kernel.  The reference resizes the frames
    of a video file in torchvision's channels-last layout and those of an image folder contiguous, and torch rounds
    the two differently; `from_video` selects which one is reproduced."""
    x = torch.from_numpy(np.ascontiguousarray(frames_bgr)).to(device)
    return ops.unpack_video_uint8(x, lr_size(x.shape[1], x.shape[2]), channels_last=from_video)


def checkpoint_paths(args: argparse.Namespace) -> dict:
    """the files inference_upscale_a_video.py:101-131 loads, checked up front so that a missing one is named"""
    d = args.model_dir
    vae = "vae_video" if args.use_video_vae else "vae_3d"
    paths = {
        "text_encoder": os.path.join(d, "text_encoder", "config.json"),
        "tokenizer": os.path.join(d, "tokenizer"),
        "low_res_scheduler": os.path.join(d, "low_res_scheduler", "scheduler_config.json"),
        "vae_config": os.path.join(d, "vae", f"{vae}_config.json"),
        "vae": os.path.join(d, "vae", f"{vae}.bin"),
        "unet_config": os.path.join(d, "unet", "unet_video_config.json"),
        "unet": os.path.join(d, "unet", "unet_video.bin"),
        "scheduler": os.path.join(d, "scheduler", "scheduler_config.json"),
    }
    if args.propagation_steps:
        paths["raft"] = os.path.join(d, "propagator", "raft-things.pth")
    for p in paths.values():
        if not os.path.exists(p):
            raise FileNotFoundError(f"missing checkpoint file: {p} (--model_dir {d})")
    return paths


def load_models(args: argparse.Namespace, paths: dict, device):
    """inference_upscale_a_video.py:100-131 from `checkpoint_paths(args)`: returns (pipeline, raft or None) on `device`"""
    from . import AutoencoderKLVideo, DDIMScheduler, Propagation, RAFT_bi, UNetVideoModel, VideoUpscalePipeline
    pipeline = VideoUpscalePipeline.from_pretrained(args.model_dir, torch_dtype=torch.float16)
    pipeline.vae = AutoencoderKLVideo.from_config(paths["vae_config"])
    pipeline.vae.load_state_dict(torch.load(paths["vae"], map_location="cpu"))
    unet = UNetVideoModel.from_config(paths["unet_config"])
    unet.load_state_dict(torch.load(paths["unet"], map_location="cpu"), strict=True)
    pipeline.unet = unet.half().eval()
    pipeline.scheduler = DDIMScheduler.from_config(paths["scheduler"])
    raft = None
    if args.propagation_steps:
        raft = RAFT_bi(paths["raft"], device=device)
        pipeline.propagator = Propagation(4, learnable=False)
    return pipeline.to(device), raft


def upscale_clip(pipeline, raft, vframes: torch.Tensor, args: argparse.Namespace, prompt: str,
                 fix_colors: bool = True) -> Iterator[Tuple[int, int, torch.Tensor]]:
    """inference_upscale_a_video.py:190-333, 3 frames at a time: samples the (1, 3, t, h, w) LR clip, then yields
    `(s, e, frames)` in time order, `frames` the colour-fixed (e - s, 3, 4h, 4w) output of frames [s, e) in [-1, 1].
    Ranks that write nothing pass `fix_colors=False` (and get the decoded (1, 3, e - s, 4h, 4w) chunks): they only
    have to take part in the collectives that run inside the iteration."""
    flows_bi = list(raft.forward_slicing(vframes)) if raft is not None else None
    _, _, _, h, w = vframes.shape
    generator = torch.Generator(device=vframes.device).manual_seed(SEED)
    kwargs = dict(num_inference_steps=args.inference_steps, guidance_scale=args.guidance_scale,
                  noise_level=args.noise_level, negative_prompt=args.n_prompt,
                  propagation_steps=args.propagation_steps)
    if args.perform_tile or tiling.needs_tiling(h, w):
        chunks = tiling.iter_upscale_tiled(pipeline, vframes, flows_bi, generator, tile_size=args.tile_size,
                                           overlap=TILE_OVERLAP, prompt=prompt, **kwargs)
    else:
        sampled = pipeline.sample_latents(prompt, image=vframes, flows_bi=flows_bi, generator=generator, **kwargs)
        chunks = pipeline.decode_chunks(sampled)
    for s, e, chunk in chunks:
        if fix_colors:
            chunk = color_correction.color_fix_frames(chunk, vframes[:, :, s:e], args.color_fix)
        yield s, e, chunk


def _init_distributed():
    """one process per GPU under torchrun: returns (device, whether this call initialised the process group)"""
    import torch.distributed as dist
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local_rank)
        dist.init_process_group(backend="nccl", device_id=torch.device("cuda", local_rank))
        return torch.device("cuda", local_rank), True
    if not torch.cuda.is_available():
        raise RuntimeError("upscale_a_video_b200 needs a CUDA GPU")
    return torch.device("cuda", torch.cuda.current_device()), False


def main(argv: Optional[List[str]] = None) -> List[str]:
    """runs the command; returns the mp4 paths written (empty on ranks other than 0)"""
    import torch.distributed as dist
    args = parse_args(argv)
    video_list = video_io.find_inputs(args.input_path)
    paths = checkpoint_paths(args)
    device, own_group = _init_distributed()
    try:
        rank = dist.get_rank() if dist.is_initialized() else 0
        log = print if rank == 0 else (lambda *a, **k: None)
        log("Loading Upscale-A-Video")
        pipeline, raft = load_models(args, paths, device)
        agent = None
        if use_llava(args) and rank == 0:
            from .llava import LLavaAgent
            log("Loading LLaVA")
            agent = LLavaAgent(args.llava_path, device=device, vision_tower_path=args.llava_vision_path,
                               weights="int8" if args.llava_int8 else "fp16")
        from .llava import CAPTION_BATCH
        captions: List[str] = []  # captions of the next clips, computed a group ahead
        written = []
        for i, video_path in enumerate(video_list):
            frames, fps, video_name = video_io.read_frames(video_path)
            index_str = f"[{i + 1}/{len(video_list)}]"
            log(f"{index_str} Processing video: ", video_name)
            caption = args.caption
            if use_llava(args):
                log(f"{index_str} Generating video caption with LLaVA...")
                if not captions:
                    captions = _shared_captions(agent, frames[0], video_list[i:i + CAPTION_BATCH], rank)
                caption = captions.pop(0)
                log(textwrap.indent(textwrap.fill("Caption: " + caption, width=80), " " * 8))
            vframes = ingest_frames(frames, device, from_video=video_io.is_video(video_path))
            video_path_out, frame_dir = output_paths(args, video_name)
            writer = None
            if rank == 0:
                os.makedirs(os.path.dirname(video_path_out), exist_ok=True)
                writer = video_io.VideoWriter(video_path_out, fps, (4 * vframes.shape[-2], 4 * vframes.shape[-1]))
            torch.cuda.synchronize(device)
            start, write_time = time.time(), 0.0
            try:
                with writer or contextlib.nullcontext():
                    for s, _, output in upscale_clip(pipeline, raft, vframes, args, caption + args.a_prompt,
                                                     fix_colors=rank == 0):
                        if writer is None:
                            continue
                        video = color_correction.pack_video_uint8(output).cpu().numpy()
                        png = color_correction.pack_frames_png(output).cpu().numpy() if args.save_image else None
                        t0 = time.time()
                        if png is not None:
                            video_io.write_frames(frame_dir, png, start=s)
                        writer.write(video)
                        write_time += time.time() - t0
                torch.cuda.synchronize(device)
            except BaseException:
                if writer is not None and os.path.exists(video_path_out):
                    os.remove(video_path_out)  # a partial mp4 would pass for a result
                raise
            run_time = time.time() - start - write_time  # GPU work and device-to-host copies, not file writing
            if rank != 0:
                continue
            written.append(video_path_out)
            log(f"{index_str} Saving upscaled video... time (sec): {run_time:.2f} \n")
        if written:
            log(f"\nAll video results are saved in {os.path.dirname(written[-1])}")
        return written
    finally:
        if own_group:
            dist.destroy_process_group()
