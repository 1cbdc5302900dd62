"""Device memory and wall time of the streaming output path against the whole-clip path, for clips of 16, 32 and 64
frames at 180x320 -> 720x1280 (synthetic weights, 2 DDIM steps with propagation at both, Wavelet colour fix).

Both paths sample with `VideoUpscalePipeline.sample_latents`.  The output phase then differs:
  * stream: per 3-frame chunk of `decode_chunks`, what `python -m upscale_a_video_b200 --save_image` does per chunk:
    `color_fix_frames`, `pack_video_uint8`, `pack_frames_png`, copies to the host;
  * whole: `torch.cat` of every chunk (what `__call__` returns), then the same steps on the whole clip.
The peak of each phase is `max_memory_allocated()` minus `memory_allocated()` where the phase starts; the run's peak is
the absolute `max_memory_allocated()`.  The growth of each phase's absolute peak between the two longest clips gives
its cost per frame, and from it the longest clip each path fits in the card's memory (a projection: nothing is run to
an out-of-memory error).  A phase whose peak at those lengths is still set by a fixed cost (the decoder's activations
for one chunk) grows faster beyond them, and its projection is optimistic.  Prints the card and its power limit;
`--out DIR` also writes DIR/measure_long_clip.json."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from upscale_a_video_b200 import color_correction  # noqa: E402

H, W, STEPS, PROP = 180, 320, 2, [0, 1]


def _sync_bytes():
    torch.cuda.synchronize()
    return torch.cuda.memory_allocated()


def run(pipe, T, path):
    image, fw, bw, pe = (x.cuda() for x in bench.synth_inputs(T, H, W, "cpu"))
    neg, pos = pe.half().chunk(2)
    kw = dict(image=image, flows_bi=[fw, bw], num_inference_steps=STEPS, guidance_scale=6.0, noise_level=120,
              prompt_embeds=pos, negative_prompt_embeds=neg, propagation_steps=PROP,
              generator=torch.Generator(device="cuda").manual_seed(10))
    start = _sync_bytes()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    sampled = pipe.sample_latents(None, **kw)
    sample_phase = torch.cuda.max_memory_allocated() - start
    mid = _sync_bytes()
    t1 = time.time()
    torch.cuda.reset_peak_memory_stats()
    n = 0
    if path == "stream":
        for s, e, chunk in pipe.decode_chunks(sampled):
            frames = color_correction.color_fix_frames(chunk, image[:, :, s:e], "Wavelet")
            n += color_correction.pack_video_uint8(frames).cpu().shape[0]
            color_correction.pack_frames_png(frames).cpu()
    else:
        output = torch.cat([f for _, _, f in pipe.decode_chunks(sampled)], dim=2)
        frames = color_correction.color_fix_frames(output, image, "Wavelet")
        del output
        n += color_correction.pack_video_uint8(frames).cpu().shape[0]
        color_correction.pack_frames_png(frames).cpu()
        del frames
    torch.cuda.synchronize()
    t2 = time.time()
    assert n == T
    output_phase = torch.cuda.max_memory_allocated() - mid
    return dict(T=T, path=path, wall_s=t2 - t0, sample_s=t1 - t0, output_s=t2 - t1, sample_phase_bytes=sample_phase,
                output_phase_bytes=output_phase, sample_peak_bytes=start + sample_phase, output_peak_bytes=mid + output_phase,
                run_peak_bytes=max(start + sample_phase, mid + output_phase))


def line(rows, key):
    """(value at 0 frames, growth per frame) of `key` through the two longest clips"""
    (t0, y0), (t1, y1) = sorted((r["T"], r[key]) for r in rows)[-2:]
    b = (y1 - y0) / (t1 - t0)
    return y1 - b * t1, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="16,32,64")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | {smi}", flush=True)
    pipe = bench.build_pipeline("cuda")
    models = _sync_bytes()
    cap = torch.cuda.get_device_properties(0).total_memory
    run(pipe, 8, "stream")  # warm-up: module loads and first launches
    run(pipe, 8, "whole")
    rows = []
    for T in [int(x) for x in args.frames.split(",")]:
        for rep in range(args.reps):
            for path in ("stream", "whole"):  # alternating
                r = run(pipe, T, path)
                r["rep"] = rep
                rows.append(r)
                print(f"T={T:3d} {path:6s} rep {rep}: wall {r['wall_s']:.2f} s (sampling {r['sample_s']:.2f}, output "
                      f"{r['output_s']:.2f}) | sampling phase {r['sample_phase_bytes'] / 2**30:.3f} GiB, output phase "
                      f"{r['output_phase_bytes'] / 2**30:.3f} GiB, run peak {r['run_peak_bytes'] / 2**30:.2f} GiB", flush=True)
    summary = {}
    for path in ("stream", "whole"):
        pts = [r for r in rows if r["path"] == path and r["rep"] == 0]
        lines = {k: line(pts, k) for k in ("sample_peak_bytes", "output_peak_bytes")}
        t_max = min((cap - a) / b if b > 0 else float("inf") for a, b in lines.values())
        summary[path] = dict(sample_peak_per_frame=lines["sample_peak_bytes"][1],
                             output_peak_per_frame=lines["output_peak_bytes"][1],
                             sample_phase_per_frame=line(pts, "sample_phase_bytes")[1],
                             output_phase_per_frame=line(pts, "output_phase_bytes")[1],
                             longest_clip_frames=int(t_max))
        m = summary[path]
        print(f"{path:6s}: per frame, sampling phase +{m['sample_phase_per_frame'] / 2**20:.2f} MiB, output phase "
              f"+{m['output_phase_per_frame'] / 2**20:.2f} MiB; absolute peaks +{m['sample_peak_per_frame'] / 2**20:.2f} / "
              f"+{m['output_peak_per_frame'] / 2**20:.2f} MiB -> longest clip within {cap / 2**30:.1f} GiB: "
              f"about {m['longest_clip_frames']} frames", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        json.dump(dict(device=smi, models_bytes=models, card_bytes=cap, rows=rows, summary=summary),
                  open(os.path.join(args.out, "measure_long_clip.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
