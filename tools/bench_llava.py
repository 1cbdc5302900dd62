"""Time the LLaVA-1.5 captioner at the 13B shape with seeded weights (CUDA events): the vision tower (CLIP ViT-L/14-336,
23 layers), the prefill of the prompt with its 576 image rows, ms per decoded token, seconds per caption of 64 new
tokens, and `uav_gemv` GB/s per decode shape against the H100 SXM data sheet's 3.35 TB/s.  When transformers is
importable, `LlamaForCausalLM.generate` (fp16, greedy, 64 new tokens) on the same weights is timed in the same run as a
baseline.  Prints the card's name and power limit first.

With `--rows 1,2,4,8`, for each row count B: `uav_gemv_rows` µs and GB/s at the five decode shapes, ms per batched
decode step (B rows, one weight pass), the prefill's ms, and seconds for one `generate_ids_batch` call captioning B
images (vision tower, prefill, 64 sampled tokens per row).  `--weights fp16,int8` builds one agent per weight format
(the int8 one quantizes each seeded matrix as it is made, so no fp16 copy of it is held), reports each agent's
`memory_allocated()`, and times the formats alternately for each row count; the int8 decoder shapes are timed on
`uav_gemv_rows_int8`, whose bytes are N K + 4 N + 2 B (K + N).

    python tools/bench_llava.py [--layers 40] [--rows 1,2,4,8] [--weights fp16,int8] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, HEADS, INTER, VOCAB = 5120, 40, 13824, 32000
VH, VHEADS, VINTER, VLAYERS = 1024, 16, 4096, 23
NEW_TOKENS = 64
HBM_TBS = 3.35


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip()


def events_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def build_agent(layers: int, weights: str = "fp16"):
    from upscale_a_video_b200 import ops
    from upscale_a_video_b200.llava import PATCH_K_PADDED, Int8Rows, LLavaAgent, dequant_scratch
    g = torch.Generator(device="cuda").manual_seed(0)
    lin = lambda a, b, s=1.0: (torch.randn(a, b, generator=g, device="cuda", dtype=torch.float16) * (s / b ** 0.5))
    if weights == "int8":
        lin16 = lin

        def lin(a, b, s=1.0):  # the agent's int8 Linears, quantized as they are made
            t = Int8Rows(torch.empty(a, b, dtype=torch.int8, device="cuda"),
                         torch.empty(a, dtype=torch.float32, device="cuda"))
            ops.quantize_rows_int8(lin16(a, b, s), t.q, t.absmax)
            return t
    vec = lambda n, c=1.0: (c + 0.1 * torch.randn(n, generator=g, device="cuda")).half()
    agent = LLavaAgent.__new__(LLavaAgent)
    agent.device = torch.device("cuda", torch.cuda.current_device())
    agent.config = SimpleNamespace(hidden_size=H, num_attention_heads=HEADS, num_hidden_layers=layers, rms_norm_eps=1e-5,
                                   rope_theta=10000.0, vocab_size=VOCAB)
    lin_fp16 = lin16 if weights == "int8" else lin
    w = {"embed": lin_fp16(VOCAB, H, H ** 0.5 * 0.02), "norm": vec(H), "lm_head": lin_fp16(VOCAB, H, 3.0),
         "proj0_w": lin(H, VH), "proj0_b": torch.zeros(H, device="cuda"), "proj2_w": lin(H, H),
         "proj2_b": torch.zeros(H, device="cuda")}
    for i in range(layers):
        w.update({f"qkv{i}": lin(3 * H, H), f"o{i}": lin(H, H), f"gu{i}": lin(2 * INTER, H), f"down{i}": lin(H, INTER),
                  f"ln1_{i}": vec(H), f"ln2_{i}": vec(H)})
    agent.w = w
    agent._dq = dequant_scratch(w, agent.device)
    f32 = lambda n, c=0.0: (c + 0.02 * torch.randn(n, generator=g, device="cuda")).float()
    vl = lambda a, b: (lin_fp16(a, b), f32(a))
    agent.vision_config = SimpleNamespace(hidden_size=VH, num_attention_heads=VHEADS, image_size=336, patch_size=14,
                                          hidden_act="quick_gelu", layer_norm_eps=1e-5)
    agent.tower = SimpleNamespace(patch_w=lin_fp16(VH, PATCH_K_PADDED), cls=vec(VH, 0.0), pos=vec(577 * VH, 0.0).view(577, VH),
                                  pre_ln=(f32(VH, 1.0), f32(VH)), layers=[
                                      SimpleNamespace(ln1=(f32(VH, 1.0), f32(VH)), qkv=vl(3 * VH, VH), out=vl(VH, VH),
                                                      ln2=(f32(VH, 1.0), f32(VH)), fc1=vl(VINTER, VH), fc2=vl(VH, VINTER))
                                      for _ in range(VLAYERS)])
    return agent


def bench_gemv():
    from upscale_a_video_b200 import ops
    rows = []
    for N, K in ((3 * H, H), (H, H), (2 * INTER, H), (H, INTER), (VOCAB, H)):
        w = torch.randn(N, K, device="cuda", dtype=torch.float16)
        x = torch.randn(K, device="cuda", dtype=torch.float16)
        out = torch.empty(N, device="cuda", dtype=torch.float16)
        for _ in range(5):
            ops.gemv(w, x, out=out)
        # one pass over several copies would hide nothing: the weight (>= 52 MB) does not fit the 50 MB L2
        ms = events_ms(lambda: ops.gemv(w, x, out=out), 200)
        gbs = N * K * 2 / (ms * 1e-3) / 1e9
        rows.append(dict(N=N, K=K, us=ms * 1e3, GBs=gbs, of_peak=gbs / (HBM_TBS * 1e3)))
        del w
    return rows


def bench_gemv_rows(rows, weights="fp16"):
    """µs and GB/s of the decode GEMV per shape; with int8 weights the decoder shapes run `uav_gemv_rows_int8` and
    lm_head (fp16 in both formats) `uav_gemv_rows`"""
    from upscale_a_video_b200 import ops
    out_rows = []
    for N, K in ((3 * H, H), (H, H), (2 * INTER, H), (H, INTER), (VOCAB, H)):
        w = torch.randn(N, K, device="cuda", dtype=torch.float16)
        x = torch.randn(rows, K, device="cuda", dtype=torch.float16)
        out = torch.empty(rows, N, device="cuda", dtype=torch.float16)
        if weights == "int8" and N != VOCAB:
            q, s = torch.empty(N, K, dtype=torch.int8, device="cuda"), torch.empty(N, device="cuda")
            ops.quantize_rows_int8(w, q, s)
            call = lambda: ops.gemv_rows_int8(q, s, x, out=out)
            nbytes = N * K + 4 * N + 2 * rows * (K + N)
        else:
            call = lambda: ops.gemv_rows(w, x, out=out)
            nbytes = N * K * 2
        for _ in range(5):
            call()
        ms = events_ms(call, 200)
        gbs = nbytes / (ms * 1e-3) / 1e9
        out_rows.append(dict(N=N, K=K, weights=weights, us=ms * 1e3, GBs=gbs, of_peak=gbs / (HBM_TBS * 1e3)))
        del w, call
    return out_rows


def bench_rows(agent, px, ids, rows, weights="fp16"):
    """decode ms per step of `rows` sequences and seconds of one caption call on `rows` images"""
    pxb = px[None].expand(rows, -1, -1, -1).contiguous()
    with torch.no_grad():
        x = agent.embed_prompt(ids, agent.vision_features(pxb))
        tok = torch.full((rows,), 29871, dtype=torch.int64, device="cuda")

        def run(max_new):
            for _ in agent._run(x, max_new, lambda step, logits: tok):
                pass

        run(2)
        prefill = events_ms(lambda: run(1), 2)
        step_ms = (events_ms(lambda: run(NEW_TOKENS), 1) - prefill) / (NEW_TOKENS - 1)
        gens = lambda: [torch.Generator().manual_seed(i) for i in range(rows)]
        seconds = caption_seconds(lambda: agent.generate_ids_batch(pxb, 0.2, 0.7, None, gens(), NEW_TOKENS))
    return dict(rows=rows, weights=weights, prefill_ms=prefill, decode_ms_per_step=step_ms, seconds_per_call=seconds,
                seconds_per_caption=[s / rows for s in seconds], gemv=bench_gemv_rows(rows, weights))


def caption_seconds(call, repeats=3):
    """host seconds of `call` (which ends with the tokens on the host), after one warm-up call, `repeats` times"""
    call()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        call()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return out


def median(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--rows", type=str, default=None, help="comma-separated row counts (1..8) of the batched decode")
    ap.add_argument("--weights", type=str, default="fp16",
                    help="comma-separated weight formats of the --rows mode (fp16, int8), timed alternately")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    from upscale_a_video_b200 import _lib
    _lib.load()
    res = dict(card=card(), layers=args.layers)
    print("card, power limit:", res["card"])
    if args.rows:
        formats = args.weights.split(",")
        assert all(f in ("fp16", "int8") for f in formats), formats
        agents = {}
        res["agent_bytes"] = {}
        for f in formats:
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            agent = build_agent(args.layers, f)
            torch.cuda.synchronize()
            res["agent_bytes"][f] = torch.cuda.memory_allocated() - before
            print(f"{f} agent: memory_allocated() {res['agent_bytes'][f] / 1e9:.2f} GB ({args.layers} layers)")
            agent.prompt_ids = lambda qs=None: [1] + list(range(100, 135)) + [-200] + list(range(200, 230))
            agent.max_new_tokens = NEW_TOKENS
            agent.eos_id = -1  # seeded weights: never stop early, every row decodes 64 tokens
            agents[f] = agent
        px = torch.randn(3, 336, 336).half()
        ids = agents[formats[0]].prompt_ids()
        res["rows"] = []
        for rows in map(int, args.rows.split(",")):
            for f in formats:
                r = bench_rows(agents[f], px, ids, rows, f)
                res["rows"].append(r)
                for gv in r["gemv"]:
                    kernel = "uav_gemv_rows_int8" if f == "int8" and gv["N"] != VOCAB else "uav_gemv_rows"
                    print(f"rows={rows} {f} {kernel:18s} N={gv['N']:6d} K={gv['K']:6d}: {gv['us']:8.1f} us  "
                          f"{gv['GBs']:7.0f} GB/s  ({100 * gv['of_peak']:.0f}% of 3.35 TB/s)")
                sc = r["seconds_per_call"]
                print(f"rows={rows} {f}: decode {r['decode_ms_per_step']:.2f} ms/step, prefill {r['prefill_ms']:.1f} ms, "
                      f"{median(sc):.3f} s per call (median of {len(sc)}, {min(sc):.3f}-{max(sc):.3f}) = "
                      f"{median(sc) / rows:.3f} s per caption")
        if args.json:
            json.dump(res, open(args.json, "w"), indent=1)
        return
    res["gemv"] = bench_gemv()
    for r in res["gemv"]:
        print(f"uav_gemv N={r['N']:6d} K={r['K']:6d}: {r['us']:8.1f} us  {r['GBs']:7.0f} GB/s  "
              f"({100 * r['of_peak']:.0f}% of 3.35 TB/s)")
    agent = build_agent(args.layers)
    weight_bytes = sum(t.numel() * t.element_size() for k, t in agent.w.items() if not k.startswith("proj"))
    res["decoder_weight_GB"] = weight_bytes / 1e9
    px = torch.randn(3, 336, 336).half()
    ids = [1] + list(range(100, 135)) + [-200] + list(range(200, 230))
    with torch.no_grad():
        for _ in range(2):
            feat = agent.vision_features(px)
        res["vision_ms"] = events_ms(lambda: agent.vision_features(px), 5)
        x = agent.embed_prompt(ids, feat)
        n = x.shape[0]
        steps = {}

        def run(max_new):  # prefill, then max_new - 1 decode steps
            agent.forward_logits(x, [29871] * (max_new - 1))

        run(2)
        res["prefill_ms"] = events_ms(lambda: run(1), 3)  # prefill + lm_head of the last row
        t_all = events_ms(lambda: run(NEW_TOKENS), 2)
        res["ms_per_token"] = (t_all - res["prefill_ms"]) / (NEW_TOKENS - 1)
        # a caption: vision tower, prefill and 64 sampled tokens, each read back to the host
        agent.prompt_ids = lambda qs=None: ids
        agent.eos_id = -1  # seeded weights: never stop early
        sc = caption_seconds(lambda: agent.generate_ids(px, 0.2, 0.7, generator=torch.Generator().manual_seed(0),
                                                        max_new_tokens=NEW_TOKENS))
        res["seconds_per_caption"] = median(sc)
        res["seconds_per_caption_runs"] = sc
        steps["n_prompt_rows"] = n
    res.update(steps)
    res["decode_GBs"] = weight_bytes / (res["ms_per_token"] * 1e-3) / 1e9
    print(f"vision tower {res['vision_ms']:.2f} ms, prefill ({n} rows) {res['prefill_ms']:.2f} ms, "
          f"decode {res['ms_per_token']:.2f} ms/token ({res['decode_GBs']:.0f} GB/s of decoder weights), "
          f"{res['seconds_per_caption']:.3f} s per caption of {NEW_TOKENS} tokens")
    try:
        res["transformers"] = bench_transformers(agent, n)
        print("transformers LlamaForCausalLM.generate fp16 (same weights, prompt of "
              f"{n} tokens, {NEW_TOKENS} new): {res['transformers']['seconds']:.3f} s")
    except ImportError as e:
        print("transformers baseline skipped:", e)
    if args.json:
        json.dump(res, open(args.json, "w"), indent=1)


def bench_transformers(agent, n):
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = agent.config
    L = cfg.num_hidden_layers
    hc = LlamaConfig(hidden_size=H, intermediate_size=INTER, num_hidden_layers=L, num_attention_heads=HEADS,
                     num_key_value_heads=HEADS, vocab_size=VOCAB, rms_norm_eps=1e-5, rope_theta=10000.0,
                     max_position_embeddings=4096, torch_dtype=torch.float16)
    with torch.device("meta"):
        m = LlamaForCausalLM(hc)
    w = agent.w
    sd = {"model.embed_tokens.weight": w["embed"], "model.norm.weight": w["norm"], "lm_head.weight": w["lm_head"]}
    for i in range(L):  # views of our fused matrices: no second copy of the weights
        p = f"model.layers.{i}."
        q, k, v = w[f"qkv{i}"].split(H)
        gate, up = w[f"gu{i}"].split(INTER)
        sd.update({p + "self_attn.q_proj.weight": q, p + "self_attn.k_proj.weight": k, p + "self_attn.v_proj.weight": v,
                   p + "self_attn.o_proj.weight": w[f"o{i}"], p + "mlp.gate_proj.weight": gate,
                   p + "mlp.up_proj.weight": up, p + "mlp.down_proj.weight": w[f"down{i}"],
                   p + "input_layernorm.weight": w[f"ln1_{i}"], p + "post_attention_layernorm.weight": w[f"ln2_{i}"]})
    m.load_state_dict(sd, assign=True, strict=False)
    m.model.rotary_emb = type(m.model.rotary_emb)(config=hc, device="cuda")  # its buffers were made on the meta device
    m = m.to("cuda").eval()
    ids = torch.randint(3, VOCAB, (1, n), device="cuda")
    kw = dict(max_new_tokens=NEW_TOKENS, min_new_tokens=NEW_TOKENS, do_sample=False, use_cache=True)
    with torch.no_grad():
        m.generate(ids, **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.generate(ids, **kw)
        torch.cuda.synchronize()
    return dict(seconds=time.perf_counter() - t0)


if __name__ == "__main__":
    main()
