// conv_io.cu — the HBM-bound tail of UNetVideoModel.forward (unet_video.py:567-569, SURVEY.md §8a rows a3/a6/a15):
//   out = conv_out( SiLU( GroupNorm(x) ) )        3x3, C = 256 -> Cout = 4, written in the reference's "b c t h w" layout
// as ONE kernel that reads x once (512 B / pixel) and writes 8-16 B / pixel.  Round 1 ran it as GroupNorm apply (read +
// write of the 256-channel tensor) + the generic implicit-GEMM tile with N = 16, K = 72 k-blocks re-read 9x from L2 (0.09 of the
// HBM roofline) + a layout-conversion kernel.
//
// Formulation: with only Cout = 4 outputs per pixel an implicit GEMM wastes the tensor core on A re-reads.  Instead
//   Y[p][tap, co] = sum_c act[p][c] * w[co][tap][c]            (one GEMM per halo pixel p: M = pixels, N = 9 * Cout, K = C)
//   out[y][x][co] = bias[co] + sum_tap Y[(y, x) + off(tap)][tap, co]   ("col2im": 9 shifted adds from shared memory)
// so every activation is read from shared memory once (mma.sync.m16n8k16, fp32 accumulate) and the shift-add touches only
// 36 floats per pixel.  GroupNorm affine + SiLU are applied on the way from global to shared memory (conv zero padding =
// zeros AFTER the activation, so out-of-image halo pixels are stored as 0).
//
// One persistent CTA per SM, 16 warps: tile = 14 x 30 output pixels -> 16 x 32 halo pixels = 32 m16 tiles (2 per warp);
// K in 4 chunks of 64 channels, double buffered in shared memory, the next chunk's global loads in flight during the
// MMAs of the current one.
#include "sampler_math.cuh"
#include "uav_common.cuh"

#include <string.h>

namespace uav {

namespace {

constexpr int CO_TH = 14, CO_TW = 30;        // output tile
constexpr int CO_HH = 16, CO_HW = 32;        // halo tile (pixels)
constexpr int CO_PIX = CO_HH * CO_HW;        // 512
constexpr int CO_THREADS = 512;
constexpr int CO_KC = 64;                    // channels per chunk
constexpr int CO_NPAD = 48;                  // 9 taps x Cout (<= 5) padded to 3 x 16
constexpr int CO_YS = 37;                    // row stride (floats) of the Y tile: odd -> conflict-free column walks
constexpr int CO_XS_BYTES = CO_PIX * CO_KC * 2;  // 64 KB per buffer
constexpr int CO_C = 256;

struct ConvOutParams {
  const __half* x;
  int64_t ld;
  int T, H, W, Cout;
  const float2* affine;  // [B][C] {scale, shift}
  const __half* w;       // [Cout][3][3][C]
  const float* bias;     // [Cout] or nullptr
  void* out;             // [B][Cout][T][H][W]
  int out_f32;
  int tiles_x, tiles_y;
  int64_t num_tiles;
  // optional fused sampler epilogue (B == 2 = the classifier-free-guidance halves of one clip, fp16 working dtype):
  //   eps = u + g (c - u)  (pipeline_upscale_a_video.py:644-645), x0 = DDIMScheduler.step_v0(eps, t, sample)
  //   (scheduling_ddim.py:383-433) with torch's per-op fp16 rounding, written as (1, Cout, T, H, W) tensors
  int fuse_cfg;
  float guidance, sa, sb, inv_sa, clip_range;
  int pred_type, clip;
  const __half* sample;  // (1, Cout, T, H, W) latents x_t
  __half* noise_pred;    // (1, Cout, T, H, W)
  __half* x0;            // (1, Cout, T, H, W)
};

__global__ void __launch_bounds__(CO_THREADS, 1)
    conv_out_fused_kernel(const ConvOutParams p) {
  extern __shared__ __align__(128) uint8_t co_smem[];
  __half* xs = reinterpret_cast<__half*>(co_smem);                      // [2][512][64], 16 B chunks XOR (row & 7)
  __half* ws = reinterpret_cast<__half*>(co_smem + 2 * CO_XS_BYTES);    // [48][256], chunks XOR (row & 7)
  float* ys = reinterpret_cast<float*>(co_smem);                        // [512][37] aliases xs after the GEMM
  float* us = reinterpret_cast<float*>(co_smem + 2 * CO_XS_BYTES + CO_NPAD * CO_C * 2);  // [TH*TW*Cout] uncond half
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntap_cols = 9 * p.Cout;

  // weights: ws[tap * Cout + co][c] = w[co][tap][c]; rows >= 9 * Cout are zero
  for (int i = tid; i < CO_NPAD * (CO_C / 8); i += CO_THREADS) {
    const int n = i / (CO_C / 8), c8 = i % (CO_C / 8);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (n < ntap_cols) {
      const int tap = n / p.Cout, co = n % p.Cout;
      v = ldg16(p.w + (static_cast<int64_t>(co) * 9 + tap) * CO_C + c8 * 8);
    }
    *reinterpret_cast<uint4*>(ws + n * CO_C + ((c8 ^ (n & 7)) << 3)) = v;
  }

  const int c8 = tid & 7;          // this thread's 16-byte channel chunk inside a 64-channel k-chunk
  const int px0 = tid >> 3;        // its halo pixels: px0 + 64 j
  // fused sampler epilogue: a work item is (frame, tile) and runs the two batch items back to back
  const int nb_per_item = p.fuse_cfg ? 2 : 1;
  for (int64_t item = blockIdx.x; item < p.num_tiles; item += gridDim.x)
  for (int bi = 0; bi < nb_per_item; ++bi) {
    const int64_t tile = item;
    const int tx = static_cast<int>(tile % p.tiles_x);
    const int ty = static_cast<int>((tile / p.tiles_x) % p.tiles_y);
    const int64_t img0 = tile / (static_cast<int64_t>(p.tiles_x) * p.tiles_y);  // fused: frame index; else b * T + t
    const int b = p.fuse_cfg ? bi : static_cast<int>(img0 / p.T);
    const int t = p.fuse_cfg ? static_cast<int>(img0) : static_cast<int>(img0 % p.T);
    const int64_t img = static_cast<int64_t>(b) * p.T + t;
    const int hy0 = ty * CO_TH - 1, hx0 = tx * CO_TW - 1;  // image coordinate of halo pixel (0, 0)
    const __half* ximg = p.x + img * p.H * p.W * p.ld;
    const float2* aff = p.affine + static_cast<int64_t>(b) * CO_C;

    uint4 pre[8];
    auto prefetch = [&](int kc) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int px = px0 + 64 * j;
        const int gy = hy0 + (px >> 5), gx = hx0 + (px & 31);
        const bool ok = gy >= 0 && gy < p.H && gx >= 0 && gx < p.W;
        pre[j] = ok ? ldg16(ximg + (static_cast<int64_t>(gy) * p.W + gx) * p.ld + kc * CO_KC + c8 * 8)
                    : make_uint4(0, 0, 0, 0);
      }
    };
    auto store_transformed = [&](int kc) {
      float sc[8], sh[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 a = __ldg(aff + kc * CO_KC + c8 * 8 + j);
        sc[j] = a.x;
        sh[j] = a.y;
      }
      __half* dst = xs + (kc & 1) * (CO_PIX * CO_KC);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int px = px0 + 64 * j;
        const int gy = hy0 + (px >> 5), gx = hx0 + (px & 31);
        const bool ok = gy >= 0 && gy < p.H && gx >= 0 && gx < p.W;
        const __half2* h = reinterpret_cast<const __half2*>(&pre[j]);
        uint4 o;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = __half22float2(h[q]);
          const float u = silu_f(fmaf(f.x, sc[2 * q], sh[2 * q]));
          const float v = silu_f(fmaf(f.y, sc[2 * q + 1], sh[2 * q + 1]));
          ow[q] = ok ? pack_half2_sat(u, v) : 0u;  // zero padding of the conv applies AFTER the activation
        }
        *reinterpret_cast<uint4*>(dst + px * CO_KC + ((c8 ^ (px & 7)) << 3)) = o;
      }
    };

    float acc[2][6][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int n = 0; n < 6; ++n) acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = 0.f;

    __syncthreads();  // previous tile's col2im finished reading ys (aliases xs); weights visible on the first tile
    prefetch(0);
#pragma unroll 1
    for (int kc = 0; kc < CO_C / CO_KC; ++kc) {
      store_transformed(kc);
      __syncthreads();
      if (kc + 1 < CO_C / CO_KC) prefetch(kc + 1);
      const __half* xb = xs + (kc & 1) * (CO_PIX * CO_KC);
#pragma unroll
      for (int ks = 0; ks < CO_KC / 16; ++ks) {
        uint32_t a[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const int row = warp * 32 + m * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
          const int chk = ks * 2 + (lane >> 4);
          ldmatrix_x4(a[m], xb + row * CO_KC + ((chk ^ (row & 7)) << 3));
        }
#pragma unroll
        for (int nb = 0; nb < 3; ++nb) {
          uint32_t bf[4];
          const int row = nb * 16 + (lane & 7) + (lane >> 4) * 8;
          const int chk = kc * 8 + ks * 2 + ((lane >> 3) & 1);
          ldmatrix_x4(bf, ws + row * CO_C + ((chk ^ (row & 7)) << 3));
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            mma16816(acc[m][nb * 2], a[m], bf[0], bf[1]);
            mma16816(acc[m][nb * 2 + 1], a[m], bf[2], bf[3]);
          }
        }
      }
    }
    __syncthreads();  // every warp is done with xs -> reuse it as the Y tile
    {
      const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < 6; ++n)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int row = warp * 32 + m * 16 + g + (e >> 1) * 8;
            const int col = n * 8 + t4 * 2 + (e & 1);
            if (col < ntap_cols) ys[row * CO_YS + col] = acc[m][n][e];
          }
    }
    __syncthreads();
    // col2im: out[y][x][co] = bias + sum over the 9 taps of Y[(y + ky, x + kx)][tap, co]
    const int64_t plane = static_cast<int64_t>(p.H) * p.W;
    for (int i = tid; i < CO_TH * CO_TW * p.Cout; i += CO_THREADS) {
      const int lx = i % CO_TW, ly = (i / CO_TW) % CO_TH, co = i / (CO_TW * CO_TH);
      const int gy = ty * CO_TH + ly, gx = tx * CO_TW + lx;
      if (gy >= p.H || gx >= p.W) continue;
      float s = p.bias != nullptr ? __ldg(p.bias + co) : 0.f;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
          s += ys[((ly + ky) * CO_HW + lx + kx) * CO_YS + (ky * 3 + kx) * p.Cout + co];
      if (p.fuse_cfg) {
        const float unet = Num<true>::rh(fminf(fmaxf(s, -65504.f), 65504.f));  // the UNet's fp16 output
        if (bi == 0) {
          us[i] = unet;  // unconditional half
        } else {
          const float eps = cfg_combine<true>(us[i], unet, p.guidance);
          const int64_t o = (static_cast<int64_t>(co) * p.T + t) * plane + static_cast<int64_t>(gy) * p.W + gx;
          const float r = ddim_x0<true>(eps, __half2float(p.sample[o]), p.pred_type, p.sa, p.sb, p.inv_sa, p.clip,
                                        p.clip_range);
          p.noise_pred[o] = __float2half_rn(eps);
          p.x0[o] = __float2half_rn(r);
        }
        continue;
      }
      const int64_t o = ((static_cast<int64_t>(b) * p.Cout + co) * p.T + t) * plane + static_cast<int64_t>(gy) * p.W + gx;
      if (p.out_f32) reinterpret_cast<float*>(p.out)[o] = s;
      else reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(fminf(fmaxf(s, -65504.f), 65504.f));
    }
  }
}

}  // namespace
}  // namespace uav

using namespace uav;

extern "C" {

static uav_status_t conv_out_launch(const void* x, int64_t B, int64_t T, int64_t H, int64_t W, int64_t C, int64_t ld,
                                    const float* affine, const void* w, const float* bias, int64_t Cout, void* out,
                                    int out_dtype, const uav_cfg_step_t* fs, cudaStream_t stream) {
  UAV_REQUIRE(x && affine && w && (out || fs), "uav_conv_out_fused: null pointer");
  UAV_REQUIRE(B > 0 && T > 0 && H > 0 && W > 0 && C == CO_C && ld >= C && ld % 8 == 0 && Cout >= 1 && Cout <= 5,
              "uav_conv_out_fused: needs C == 256 input channels and 1..5 output channels (C=%lld Cout=%lld)",
              (long long)C, (long long)Cout);
  UAV_REQUIRE_ALIGNED16("uav_conv_out_fused", x);
  UAV_REQUIRE_ALIGNED16("uav_conv_out_fused", w);
  UAV_REQUIRE(out_dtype == UAV_F16 || out_dtype == UAV_F32, "uav_conv_out_fused: bad out_dtype");
  ConvOutParams p;
  memset(&p, 0, sizeof(p));
  p.x = reinterpret_cast<const __half*>(x);
  p.ld = ld;
  p.T = (int)T;
  p.H = (int)H;
  p.W = (int)W;
  p.Cout = (int)Cout;
  p.affine = reinterpret_cast<const float2*>(affine);
  p.w = reinterpret_cast<const __half*>(w);
  p.bias = bias;
  p.out = out;
  p.out_f32 = out_dtype == UAV_F32;
  p.tiles_x = (int)((W + CO_TW - 1) / CO_TW);
  p.tiles_y = (int)((H + CO_TH - 1) / CO_TH);
  p.num_tiles = (int64_t)p.tiles_x * p.tiles_y * B * T;
  if (fs != nullptr) {
    UAV_REQUIRE(B == 2 && fs->sample && fs->noise_pred && fs->pred_original_sample && fs->pred_type >= 0 &&
                    fs->pred_type <= 2 && fs->sqrt_alpha > 0.f,
                "uav_conv_out_cfg_step: needs the two guidance halves (B == 2) and sample / noise_pred / x0 tensors");
    p.fuse_cfg = 1;
    p.num_tiles = (int64_t)p.tiles_x * p.tiles_y * T;
    p.guidance = fs->guidance_scale;
    p.sa = fs->sqrt_alpha;
    p.sb = fs->sqrt_beta;
    p.inv_sa = 1.0f / fs->sqrt_alpha;
    p.pred_type = fs->pred_type;
    p.clip = fs->clip;
    p.clip_range = fs->clip_range;
    p.sample = reinterpret_cast<const __half*>(fs->sample);
    p.noise_pred = reinterpret_cast<__half*>(fs->noise_pred);
    p.x0 = reinterpret_cast<__half*>(fs->pred_original_sample);
  }
  constexpr int SMEM = 2 * CO_XS_BYTES + CO_NPAD * CO_C * 2 + CO_TH * CO_TW * 5 * 4;
  static_assert(CO_PIX * CO_YS * 4 <= 2 * CO_XS_BYTES, "Y tile must fit in the activation buffers");
  int64_t grid = num_sms();
  if (grid > p.num_tiles) grid = p.num_tiles;
  return launch_opted_in<conv_out_fused_kernel>((unsigned)grid, CO_THREADS, SMEM, stream, p);
}

uav_status_t uav_conv_out_fused(const void* x, int64_t B, int64_t T, int64_t H, int64_t W, int64_t C, int64_t ld,
                                const float* affine, const void* w, const float* bias, int64_t Cout, void* out,
                                int out_dtype, uav_stream_t stream) {
  return conv_out_launch(x, B, T, H, W, C, ld, affine, w, bias, Cout, out, out_dtype, nullptr, (cudaStream_t)stream);
}

uav_status_t uav_conv_out_cfg_step(const void* x, int64_t T, int64_t H, int64_t W, int64_t C, int64_t ld,
                                   const float* affine, const void* w, const float* bias, int64_t Cout,
                                   const uav_cfg_step_t* step, uav_stream_t stream) {
  UAV_REQUIRE(step != nullptr, "uav_conv_out_cfg_step: null step descriptor");
  return conv_out_launch(x, 2, T, H, W, C, ld, affine, w, bias, Cout, nullptr, UAV_F16, step, (cudaStream_t)stream);
}

}  // extern "C"
