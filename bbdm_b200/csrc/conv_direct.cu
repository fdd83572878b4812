// General fp32 convolution on CUDA cores (SIMT implicit GEMM, 64 pixels x TN couts per CTA).
// Serves the UNet edges (stem Cin=3..32, head Cout=3..16), conv-mode Down/Upsample and any
// channel count the wgmma kernel does not take.  fp32 FMA accumulation, two-level: each 16-channel chunk of a tap is
// summed on its own and then added to the output's total, so the rounding error grows with Cin / 16 + k*k*Cin / 16
// additions instead of k*k*Cin (a 3x3 conv over 1024 channels sums 9216 products).
#include "common.cuh"

namespace bbdm {

constexpr int CD_TM = 64;   // output pixels per CTA
constexpr int CD_TK = 16;   // cin chunk

template <int TN>           // couts per CTA: 64 or 16
__global__ void __launch_bounds__(256)
conv_direct_kernel(const float* __restrict__ src, const float* __restrict__ wp,
                   const float* __restrict__ bias, const float* __restrict__ res,
                   float* __restrict__ out, int B, int H, int W, int Cin, int Cout, int k,
                   int stride, int Ho, int Wo, int pad) {
  constexpr int TPN = TN / 4;          // threads along N (each 4 couts)
  constexpr int TPM = 256 / TPN;       // threads along M
  constexpr int PM = CD_TM / TPM;      // pixels per thread (TN=64: 4 ; TN=16: 1)
  __shared__ float As[CD_TK][CD_TM + 4];
  __shared__ float Ws[CD_TK][TN + 4];
  const int tid = threadIdx.x;
  const int tn = tid % TPN, tm = tid / TPN;
  const int64_t M = (int64_t)B * Ho * Wo;
  const int64_t m0 = (int64_t)blockIdx.x * CD_TM;
  const int n0 = blockIdx.y * TN;

  // A-load assignment: 64 pixels x 16 cin = 1024 elements, 4 per thread
  const int a_p = tid / 4;             // pixel within tile
  const int a_k = (tid % 4) * 4;       // first cin within chunk
  int ab = 0, aho = 0, awo = 0;
  const bool a_valid = (m0 + a_p) < M;
  if (a_valid) {
    int64_t m = m0 + a_p;
    awo = (int)(m % Wo); m /= Wo;
    aho = (int)(m % Ho);
    ab = (int)(m / Ho);
  }
  float acc[PM][4];
#pragma unroll
  for (int i = 0; i < PM; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int tap = 0; tap < k * k; ++tap) {
    const int dy = tap / k - pad, dx = tap % k - pad;
    const int hi = aho * stride + dy, wi = awo * stride + dx;
    const bool in_img = a_valid && hi >= 0 && hi < H && wi >= 0 && wi < W;
    const float* arow = src + (((int64_t)ab * H + hi) * W + wi) * Cin;
    for (int c0 = 0; c0 < Cin; c0 += CD_TK) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c0 + a_k + j;
        As[a_k + j][a_p] = (in_img && c < Cin) ? arow[c] : 0.f;
      }
      // W tile: 16 x TN
      for (int i = tid; i < CD_TK * TN; i += 256) {
        const int kk = i / TN, n = i % TN;
        const int c = c0 + kk, co = n0 + n;
        Ws[kk][n] = (c < Cin && co < Cout) ? wp[((int64_t)tap * Cin + c) * Cout + co] : 0.f;
      }
      __syncthreads();
      float part[PM][4];
#pragma unroll
      for (int i = 0; i < PM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) part[i][j] = 0.f;
#pragma unroll
      for (int kk = 0; kk < CD_TK; ++kk) {
        float a[PM], w[4];
#pragma unroll
        for (int i = 0; i < PM; ++i) a[i] = As[kk][tm * PM + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = Ws[kk][tn * 4 + j];
#pragma unroll
        for (int i = 0; i < PM; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) part[i][j] = fmaf(a[i], w[j], part[i][j]);
      }
#pragma unroll
      for (int i = 0; i < PM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += part[i][j];
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < PM; ++i) {
    const int64_t m = m0 + tm * PM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = n0 + tn * 4 + j;
      if (co >= Cout) continue;
      float v = acc[i][j] + (bias ? bias[co] : 0.f);
      if (res) v += res[m * Cout + co];
      out[m * Cout + co] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// UNet stem (openaimodel.py:524: Conv2d(in_channels, model_channels, 3, padding=1), Cin = 3..16): the general kernel
// above pads its 16-channel K chunk with zeros (62 % wasted at Cin = 6) and synchronises per tap -- 1.35 ms at cfg2.
// Here one CTA owns one image row: the whole weight set (<= 9*16*128 floats) sits in shared memory, the 3-row input
// strip of a 32-pixel sub-tile is staged once, lane l accumulates couts l, l+32, .. for 4 pixels, and the row's
// GroupNorm partial sums (sum, sum of squares per cout) come out of the same pass (the separate statistics pass over
// the stem output disappears).  Same fp32 FMA order as conv_direct_kernel (tap-major, channel-minor) => identical bits.
template <int NJ>            // couts per lane: Cout / 32 (1..4)
__global__ void __launch_bounds__(256)
conv_stem_kernel(const float* __restrict__ src, const float* __restrict__ wp, const float* __restrict__ bias,
                 float* __restrict__ out, int H, int W, int Cin, float* __restrict__ stats) {
  extern __shared__ float sm[];
  const int Cout = NJ * 32;
  float* ws = sm;                                   // [9*Cin][Cout]
  float* as = sm + 9 * Cin * Cout;                  // [3][34][Cin]
  float* red = as + 3 * 34 * Cin;                   // [8][Cout][2]
  const int b = blockIdx.x / H, y = blockIdx.x % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 9 * Cin * Cout; i += 256) ws[i] = wp[i];
  float bj[NJ], ssum[NJ], ssq[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) { bj[j] = bias ? bias[lane + 32 * j] : 0.f; ssum[j] = 0.f; ssq[j] = 0.f; }
  for (int x0 = 0; x0 < W; x0 += 32) {
    __syncthreads();                                // previous sub-tile done with `as` (and ws loaded)
    for (int i = threadIdx.x; i < 3 * 34 * Cin; i += 256) {
      const int c = i % Cin, col = (i / Cin) % 34, r = i / (Cin * 34);
      const int yy = y + r - 1, xx = x0 + col - 1;
      as[i] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? src[(((int64_t)b * H + yy) * W + xx) * Cin + c] : 0.f;
    }
    __syncthreads();
    float acc[4][NJ];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3, dx = tap % 3;
      const float* arow = as + (dy * 34 + warp * 4 + dx) * Cin;
      const float* wrow = ws + tap * Cin * Cout + lane;
      // the general kernel's two-level order (Cin <= 16 is one chunk per tap): bit-identical results
      float part[4][NJ];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) part[i][j] = 0.f;
      for (int c = 0; c < Cin; ++c) {
        float w[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) w[j] = wrow[c * Cout + 32 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float a = arow[i * Cin + c];
#pragma unroll
          for (int j = 0; j < NJ; ++j) part[i][j] = fmaf(a, w[j], part[i][j]);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] += part[i][j];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = x0 + warp * 4 + i;
      float* o = out + (((int64_t)b * H + y) * W + x) * Cout + lane;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float v = acc[i][j] + bj[j];
        o[32 * j] = v;
        ssum[j] += v;
        ssq[j] = fmaf(v, v, ssq[j]);
      }
    }
  }
  if (stats) {
    // fixed-order combine of the 8 warps => deterministic partial sums, one row per image row
#pragma unroll
    for (int j = 0; j < NJ; ++j) { red[(warp * Cout + lane + 32 * j) * 2] = ssum[j]; red[(warp * Cout + lane + 32 * j) * 2 + 1] = ssq[j]; }
    __syncthreads();
    for (int c = threadIdx.x; c < Cout; c += 256) {
      float a = 0.f, q = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) { a += red[(k * Cout + c) * 2]; q += red[(k * Cout + c) * 2 + 1]; }
      *reinterpret_cast<float2*>(stats + ((int64_t)blockIdx.x * Cout + c) * 2) = make_float2(a, q);
    }
  }
}

}  // namespace bbdm

using namespace bbdm;

static int conv_direct_launch(const float* src, const float* w_packed, const float* bias, const float* residual,
                              float* out, int B, int H, int W, int Cin, int Cout, int k, int stride, int pad_lo,
                              int pad_hi, void* stream) {
  BBDM_REQUIRE(src && w_packed && out, "conv_direct: null pointer");
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && (k == 1 || k == 3) && (stride == 1 || stride == 2) &&
               pad_lo >= 0 && pad_hi >= 0 && pad_lo < k && pad_hi < k, "conv_direct: bad shape");
  BBDM_REQUIRE(H + pad_lo + pad_hi >= k && W + pad_lo + pad_hi >= k, "conv_direct: input smaller than the kernel");
  const int Ho = (H + pad_lo + pad_hi - k) / stride + 1, Wo = (W + pad_lo + pad_hi - k) / stride + 1;
  const int64_t M = (int64_t)B * Ho * Wo;
  const int64_t gm = (M + CD_TM - 1) / CD_TM;
  BBDM_REQUIRE(gm < (1ll << 31), "conv_direct: too many pixels");
  cudaStream_t s = (cudaStream_t)stream;
  if (Cout <= 16) {
    dim3 grid((unsigned)gm, (Cout + 15) / 16);
    conv_direct_kernel<16><<<grid, 256, 0, s>>>(src, w_packed, bias, residual, out, B, H, W, Cin, Cout, k, stride, Ho, Wo, pad_lo);
  } else {
    dim3 grid((unsigned)gm, (Cout + 63) / 64);
    conv_direct_kernel<64><<<grid, 256, 0, s>>>(src, w_packed, bias, residual, out, B, H, W, Cin, Cout, k, stride, Ho, Wo, pad_lo);
  }
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

extern "C" int bbdm_conv_direct(const float* src, const float* w_packed, const float* bias,
                                const float* residual, float* out, int B, int H, int W, int Cin,
                                int Cout, int k, int stride, void* stream) {
  return conv_direct_launch(src, w_packed, bias, residual, out, B, H, W, Cin, Cout, k, stride, k / 2, k / 2, stream);
}

// explicit zero padding: pad_lo rows/cols before, pad_hi after (VQGAN Downsample pads (0,1,0,1) and strides by
// 2 with no further padding, model/VQGAN/model.py:55-73).  out: [B, Ho, Wo, Cout], Ho = (H+pad_lo+pad_hi-k)/stride+1
extern "C" int bbdm_conv_direct_pad(const float* src, const float* w_packed, const float* bias,
                                    const float* residual, float* out, int B, int H, int W, int Cin,
                                    int Cout, int k, int stride, int pad_lo, int pad_hi, void* stream) {
  return conv_direct_launch(src, w_packed, bias, residual, out, B, H, W, Cin, Cout, k, stride, pad_lo, pad_hi, stream);
}

// ---------------------------------------------------------------------------------------------
// Weight gradient for the small-channel convolutions (UNet stem Cin = 3..32, head Cout = 3..16):
//   dW[tap][co][ci] = sum_p dY[p][co] * X[p + tap][ci]          fp32 FMA, stride 1, pad k/2
// One CTA per chunk of pixels and chunk of 1024 (co, ci) pairs (grid y); thread t owns the pairs t, t+256, ... of its
// chunk for all taps (<= 4 pairs x 9 taps accumulators); partials [chunk][tap][Cout][Cin] are reduced in a fixed order
// by bbdm's wgrad reduce kernel (deterministic).  The work is tiny (<= 2 GFLOP) -- this kernel only
// has to not be slow; cuDNN's fp32 wgrad took 1.3 ms per call on these shapes.
// ---------------------------------------------------------------------------------------------
namespace bbdm {

constexpr int WD_MAX_PAIRS = 4;

template <int k>
__global__ void __launch_bounds__(256)
conv_wgrad_direct_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ part,
                         int B, int H, int W, int Cin, int Cout, int px_per_block) {
  const int pairs = Cin * Cout;
  constexpr int pad = k / 2, taps = k * k;
  float acc[WD_MAX_PAIRS][9];
#pragma unroll
  for (int i = 0; i < WD_MAX_PAIRS; ++i)
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[i][t] = 0.f;
  const int64_t P = (int64_t)B * H * W;
  const int64_t p0 = (int64_t)blockIdx.x * px_per_block;
  const int64_t p1 = p0 + px_per_block < P ? p0 + px_per_block : P;
  // per-thread constants of its (co, ci) pairs; pixel coordinates advance incrementally (no div/mod per pixel)
  int co_[WD_MAX_PAIRS], ci_[WD_MAX_PAIRS];
#pragma unroll
  for (int i = 0; i < WD_MAX_PAIRS; ++i) {
    const int pr = blockIdx.y * 256 * WD_MAX_PAIRS + threadIdx.x + i * 256;
    co_[i] = pr < pairs ? pr / Cin : -1;
    ci_[i] = pr < pairs ? pr % Cin : 0;
  }
  int w = (int)(p0 % W), h = (int)((p0 / W) % H);
  const float* dyp = dy + p0 * Cout;
  const float* xp = x + p0 * Cin;           // pixel p itself; neighbours are +-(W*Cin), +-Cin away inside the image
  for (int64_t p = p0; p < p1; ++p) {
    bool okh[3], okw[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      okh[d] = (unsigned)(h + d - pad) < (unsigned)H;
      okw[d] = (unsigned)(w + d - pad) < (unsigned)W;
    }
#pragma unroll
    for (int i = 0; i < WD_MAX_PAIRS; ++i) {
      if (co_[i] < 0) continue;
      const float g = dyp[co_[i]];
      const float* xc = xp + ci_[i];
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        if (t < taps) {
          constexpr int kk = k;
          const int dh = t / kk, dw = t % kk;           // compile-time after unrolling
          if (okh[dh] && okw[dw])
            acc[i][t] = fmaf(g, xc[((int64_t)(dh - pad) * W + (dw - pad)) * Cin], acc[i][t]);
        }
      }
    }
    dyp += Cout; xp += Cin;
    if (++w == W) { w = 0; if (++h == H) h = 0; }
  }
  float* o = part + (int64_t)blockIdx.x * taps * pairs;
#pragma unroll
  for (int i = 0; i < WD_MAX_PAIRS; ++i) {
    const int pr = blockIdx.y * 256 * WD_MAX_PAIRS + threadIdx.x + i * 256;
    if (pr >= pairs) continue;
#pragma unroll
    for (int t = 0; t < 9; ++t)
      if (t < taps) o[(int64_t)t * pairs + pr] = acc[i][t];                   // [tap][co][ci]
  }
}

// one warp per output element: lanes stride over the partial blocks, fixed-order shuffle tree (fp64)
__global__ void __launch_bounds__(256)
wgrad_direct_reduce_kernel(const float* __restrict__ part, int nblk, int taps, int Cout, int Cin, float* __restrict__ dw) {
  const int64_t n = (int64_t)taps * Cout * Cin;
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  double s = 0.0;
  for (int kblk = lane; kblk < nblk; kblk += 32) s += (double)part[(int64_t)kblk * n + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const int ci = (int)(i % Cin);
    const int co = (int)((i / Cin) % Cout);
    const int tap = (int)(i / ((int64_t)Cin * Cout));
    dw[((int64_t)co * Cin + ci) * taps + tap] = (float)s;
  }
}

}  // namespace bbdm

extern "C" int bbdm_conv_wgrad_direct(const float* dy, const float* x, int B, int H, int W, int Cin, int Cout, int k,
                                      float* dw, float* workspace, int64_t workspace_floats, void* stream) {
  BBDM_REQUIRE(dy && x && dw && workspace, "conv_wgrad_direct: null pointer");
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0 && (k == 1 || k == 3), "conv_wgrad_direct: bad shape");
  BBDM_REQUIRE((int64_t)Cin * Cout <= (1 << 24), "conv_wgrad_direct: Cin*Cout = %lld too large",
               (long long)Cin * Cout);
  const int64_t P = (int64_t)B * H * W;
  const int64_t n = (int64_t)k * k * Cin * Cout;
  int64_t nblk = workspace_floats / n;
  if (nblk > 4096) nblk = 4096;
  if (nblk > P) nblk = P;
  BBDM_REQUIRE(nblk >= 1, "conv_wgrad_direct: workspace too small (need >= %lld floats)", (long long)n);
  const int ppb = (int)((P + nblk - 1) / nblk);
  nblk = (P + ppb - 1) / ppb;
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)nblk, (unsigned)((Cin * Cout + 256 * bbdm::WD_MAX_PAIRS - 1) / (256 * bbdm::WD_MAX_PAIRS)));
  if (k == 3) bbdm::conv_wgrad_direct_kernel<3><<<grid, 256, 0, s>>>(dy, x, workspace, B, H, W, Cin, Cout, ppb);
  else bbdm::conv_wgrad_direct_kernel<1><<<grid, 256, 0, s>>>(dy, x, workspace, B, H, W, Cin, Cout, ppb);
  BBDM_LAUNCH_CHECK();
  bbdm::wgrad_direct_reduce_kernel<<<(unsigned)((n + 7) / 8), 256, 0, s>>>(workspace, (int)nblk, k * k, Cout, Cin, dw);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

// UNet stem: src [B,H,W,Cin] fp32 (Cin <= 16), w_packed [9][Cin][Cout] from bbdm_pack_weight_f32, k = 3, stride 1,
// pad 1, Cout in {32, 64, 96, 128}, W a multiple of 32.  stats_partial (optional): [B*H][Cout][2] GroupNorm partial
// sums of the output (rows_per_image = H for bbdm_gn_finalize_partials).
extern "C" int bbdm_conv_stem(const float* src, const float* w_packed, const float* bias, float* out, int B, int H,
                              int W, int Cin, int Cout, float* stats_partial, void* stream) {
  BBDM_REQUIRE(src && w_packed && out, "conv_stem: null pointer");
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0 && W % 32 == 0 && Cin > 0 && Cin <= 16 && Cout >= 32 && Cout <= 128 && Cout % 32 == 0,
               "conv_stem: need W %% 32 == 0, Cin <= 16, Cout in {32,64,96,128} (got W=%d Cin=%d Cout=%d)", W, Cin, Cout);
  BBDM_REQUIRE((int64_t)B * H < (1ll << 31), "conv_stem: too many rows");
  const size_t smem = ((size_t)9 * Cin * Cout + 3 * 34 * Cin + 8 * Cout * 2) * sizeof(float);
  const unsigned grid = (unsigned)((int64_t)B * H);
  cudaStream_t s = (cudaStream_t)stream;
#define BBDM_STEM(NJ)                                                                                         \
  {                                                                                                           \
    static DeviceOnce cfgd;                                                                                   \
    if (smem > 48 * 1024 && cfgd.need()) {                                                                    \
      BBDM_CUDA_CHECK(cudaFuncSetAttribute(conv_stem_kernel<NJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)); \
      cfgd.mark();                                                                                            \
    }                                                                                                         \
    conv_stem_kernel<NJ><<<grid, 256, smem, s>>>(src, w_packed, bias, out, H, W, Cin, stats_partial);          \
  }
  switch (Cout / 32) {
    case 1: BBDM_STEM(1) break;
    case 2: BBDM_STEM(2) break;
    case 3: BBDM_STEM(3) break;
    default: BBDM_STEM(4) break;
  }
#undef BBDM_STEM
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

