/*
 * bbdm_b200.h -- C ABI of the H100-native (sm_90a) BBDM hot path.
 *
 * The reference (xuekt98/BBDM) is pure Python/PyTorch: it has no FFI layer.  Its "plugin
 * boundary" for this path is the Python class contract consumed by the runner.  This header is the boundary *below* that contract: every device computation the
 * drop-in classes perform goes through exactly these entry points (bound with ctypes in
 * bbdm_b200/cabi.py).  Each entry point cites the reference code it replaces
 * (paths relative to the upstream repository).
 *
 * Conventions
 *   - plain pointers + sizes only; all pointers are DEVICE pointers unless noted
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous and
 *     stream-ordered, allocates nothing, and is CUDA-graph capturable
 *   - return 0 on success, a negative BBDM_E_* code otherwise; bbdm_last_error() returns a
 *     thread-local message; no exceptions cross the boundary
 *   - activations inside the UNet are NHWC fp32 ("[B,H,W,C]"); tensor-core operands are the
 *     same tensors split into two bf16 planes  hi = bf16(x), lo = bf16(x - hi)
 */
#ifndef BBDM_B200_H_
#define BBDM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BBDM_ABI_VERSION 11

enum {
  BBDM_OK = 0,
  BBDM_E_INVALID = -1,     /* bad argument / unsupported shape            */
  BBDM_E_CUDA = -2,        /* a CUDA runtime/driver call failed           */
  BBDM_E_UNSUPPORTED = -3, /* valid request this build cannot serve       */
  BBDM_E_DEVICE = -4       /* a kernel reported an internal fault/timeout */
};

int bbdm_abi_version(void);
const char* bbdm_last_error(void);
/* Fills sm count / compute capability of the current device; 0 on success. */
int bbdm_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* Reads (and clears) the device-side fault word written by kernels whose mbarrier waits
 * timed out, by a timestep index out of range (0xB...) or by a Winograd F(6x6,3x3) input transform
 * that left the fp16 range (0xC...); synchronises `stream`.  0 = no fault. */
int bbdm_check_device_fault(void* stream, unsigned long long* fault_word);

/* ------------------------------------------------------------------------------------------
 * Brownian-bridge elementwise kernels (NCHW fp32, any contiguous [B, n_per_sample])
 * ------------------------------------------------------------------------------------------ */

enum { BBDM_OBJ_GRAD = 0, BBDM_OBJ_NOISE = 1, BBDM_OBJ_YSUBX = 2 };

/* q_sample: x_t = (1-m_t) x0 + m_t y + sqrt(var_t) noise, plus the training objective.
 * Replaces BrownianBridgeModel.q_sample (model/BrownianBridge/BrownianBridgeModel.py:128-146)
 * and extract() (model/utils.py:4-7).  t: int64 [B]; m_t/variance_t: fp32 [T] schedule buffers.
 * Same fp32 operation order as the reference => bit-exact. */
int bbdm_bridge_q_sample(const float* x0, const float* y, const float* noise, const int64_t* t,
                         const float* m_t, const float* variance_t, int num_timesteps,
                         int objective, float* x_t_out, float* objective_out,
                         int B, int64_t n_per_sample, void* stream);

/* Per-step scalar coefficients of the reverse bridge update (host computes them in fp32 with
 * the reference's expression order; BrownianBridgeModel.py:190-199). */
typedef struct {
  float m_t, one_minus_m_t, sqrt_var_t; /* for predict_x0 (objective 'noise')      */
  float m_nt, one_minus_m_nt;           /* next-step bridge weights                */
  float c_xt;                           /* sqrt((var_nt - sigma2_t) / var_t)       */
  float sigma_t;                        /* sqrt(sigma2_t) * eta                    */
} BbdmPSampleCoef;

/* p_sample update: x0_recon = predict_x0(x_t, y, eps) [clamp], then either return x0_recon
 * (is_last) or the posterior mean + sigma_t * noise.
 * Replaces predict_x0_from_objective + the tail of p_sample
 * (BrownianBridgeModel.py:148-160, 171-201).  x0_out may be NULL. noise may be NULL iff is_last. */
int bbdm_bridge_p_sample(const float* x_t, const float* y, const float* eps, const float* noise,
                         BbdmPSampleCoef coef, int objective, int clip_denoised, int is_last,
                         float* x_out, float* x0_out, int64_t n, void* stream);

/* Same, with the coefficient struct read from DEVICE memory at kernel start, so one captured
 * CUDA graph of (UNet forward + this update) serves every non-final step of p_sample_loop
 * (BrownianBridgeModel.py:203-221): the host only rewrites 7 floats + the timestep per step. */
int bbdm_bridge_p_sample_dev(const float* x_t, const float* y, const float* eps, const float* noise,
                             const BbdmPSampleCoef* coef_dev, int objective, int clip_denoised,
                             int is_last, float* x_out, float* x0_out, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------
 * Layout / small dense ops
 * ------------------------------------------------------------------------------------------ */

/* NCHW x [B,c1,H,W] (+ NCHW ctx [B,c2,H,W], may be NULL) -> NHWC [B,H,W,c1+c2].
 * Replaces th.cat([x, context], dim=1) at openaimodel.py:741-742 + the layout change. */
int bbdm_nchw_to_nhwc_cat(const float* x, int c1, const float* ctx, int c2, int B, int H, int W,
                          float* out, void* stream);
int bbdm_nhwc_to_nchw(const float* src, int B, int H, int W, int C, float* out, void* stream);

/* out[b,:] = table[idx[b],:]  (timestep-embedding table lookup; table built on the host with
 * the reference's own expression, util.py:151-171, so indexing is bit-exact). */
int bbdm_gather_rows(const float* table, int rows, int width, const int64_t* idx, int B,
                     float* out, void* stream);

/* out[B,N] = act_in(x)[B,K] @ w[N,K]^T + bias[N]; act_in: 0 none, 1 SiLU; act_out likewise.
 * fp32 FMA on CUDA cores.  Replaces time_embed (openaimodel.py:511-516) and every
 * ResBlock.emb_layers (openaimodel.py:221-227; all 21 concatenated into one call). */
int bbdm_linear_f32(const float* x, const float* w, const float* bias, float* out,
                    int B, int K, int N, int act_in, int act_out, void* stream);

/* ------------------------------------------------------------------------------------------
 * GroupNorm statistics and the fused "operand preparation" pass
 * ------------------------------------------------------------------------------------------ */

/* mean/rstd [B,groups] over the channel-concatenation of src1 [B,H,W,c1] and src2 [B,H,W,c2]
 * (src2 may be NULL), biased variance, rstd = 1/sqrt(var+eps).
 * Replaces the statistics half of GroupNorm32 (util.py:199-216; nn.GroupNorm(32,C), eps 1e-5).
 * fp64 accumulation, fixed reduction order (run-to-run deterministic).
 * workspace: >= B*groups*BBDM_GN_MAX_SLICES*2 doubles. */
#define BBDM_GN_MAX_SLICES 64
int bbdm_gn_stats(const float* src1, int c1, const float* src2, int c2, int B, int H, int W,
                  int groups, float eps, float* mean, float* rstd, double* workspace,
                  void* stream);

enum { BBDM_RESAMPLE_NONE = 0, BBDM_RESAMPLE_UP2 = 1, BBDM_RESAMPLE_DOWN2 = 2 };

/* One pass over cat(src1, src2) [B,Hs,Ws,C] producing up to two results at the resampled
 * size [B,H,W,C]:
 *   act = resample( silu?( GN_affine(x) * (1+film_scale) + film_shift ) )
 *   raw = resample( x )
 * each as fp32 and/or as a split-bf16 pair.  mean == NULL skips the "act" result.
 * Replaces: GroupNorm affine + SiLU (openaimodel.py:205-206,229-230,688-689), the FiLM
 * scale-shift (:270-274), h_upd/x_upd = Upsample/Downsample without conv (:212-217, 93-163)
 * and th.cat([h, hs.pop()], 1) (:752). */
typedef struct {
  const float* src1; int c1;
  const float* src2; int c2;
  int B, Hs, Ws;
  int groups;
  const float* mean;         /* [B,groups] or NULL */
  const float* rstd;
  const float* gamma;        /* [C] */
  const float* beta;         /* [C] */
  const float* film_scale;   /* row b at film_scale + b*film_stride, [C]; NULL = no FiLM */
  const float* film_shift;
  int64_t film_stride;
  int silu;
  int resample;
  float* act_f32; void* act_hi; void* act_lo;   /* any may be NULL */
  float* raw_f32; void* raw_hi; void* raw_lo;
} BbdmPrepArgs;
int bbdm_prep_operand(const BbdmPrepArgs* a, void* stream);

/* ------------------------------------------------------------------------------------------
 * Convolutions
 * ------------------------------------------------------------------------------------------ */

/* Weight repacking (derived caches; the nn.Parameter stays OIHW fp32 so checkpoints/EMA are
 * unchanged).  w: [Cout,Cin,k,k] fp32 (k = 1 or 3).
 *   split:  hi/lo bf16 [k*k][Cout][Cin]   (K-major B operand of the tensor-core kernel)
 *   f32:    fp32 [k*k][Cin][Cout]         (direct kernel) */
int bbdm_pack_weight_split(const float* w, int Cout, int Cin, int k, void* w_hi, void* w_lo,
                           void* stream);
/* Same, into planes of Cout_pad >= Cout rows per tap (rows >= Cout must be pre-zeroed by the
 * caller): lets a conv with few output channels (the UNet head, Cout = 3..16) use the
 * tensor-core kernel with an N tile of 64. */
int bbdm_pack_weight_split_padded(const float* w, int Cout, int Cin, int k, int Cout_pad,
                                  void* w_hi, void* w_lo, void* stream);
/* General tap count: w [Cout][Cin][taps] fp32 -> hi/lo bf16 [taps][Cout][Cin] (used for the 16
 * phase taps of the fused-upsample conv, BbdmConvArgs.upsample2x). */
int bbdm_pack_weight_split_taps(const float* w, int Cout, int Cin, int taps, void* w_hi, void* w_lo,
                                void* stream);
/* Data-gradient planes straight from OIHW: hi/lo [k*k][Cin][Cout], kernel flipped and Cin/Cout
 * swapped, so that dX = bbdm_conv_umma(dY planes, these planes) (training backward). */
int bbdm_pack_weight_split_dgrad(const float* w, int Cout, int Cin, int k, void* w_hi, void* w_lo,
                                 void* stream);

/* Both layouts in ONE pass over the OIHW weight (the training step re-packs every weight after each optimizer
 * update): fwd_* = bbdm_pack_weight_split's planes, dgrad_* = bbdm_pack_weight_split_dgrad's; either pair may be NULL.
 * Shared-memory tiled transpose: coalesced reads and writes (the single-layout packers gather with a 36-byte stride). */
int bbdm_pack_weight_split_both(const float* w, int Cout, int Cin, int k, void* fwd_hi, void* fwd_lo, void* dgrad_hi,
                                void* dgrad_lo, void* stream);
int bbdm_pack_weight_f32(const float* w, int Cout, int Cin, int k, float* out, void* stream);

enum { BBDM_RES_NONE = 0, BBDM_RES_SAME = 1, BBDM_RES_UP2 = 2, BBDM_RES_DOWN2 = 3 };

/* Stride-1 "same" convolution as an implicit GEMM on wgmma tensor cores:
 *   out[b,h,w,:] = sum_taps A[b,h+dy,w+dx,:] . W[tap] + bias
 *                  (+ A2[b,h,w,:] . W2 + bias2)            fused 1x1 skip conv
 *                  (+ residual, optionally nearest-up / 2x2-avg resampled)
 * M = B*H*W (tile 128 = box of pixels), N = Cout, K = taps*Cin (+ Cin2); operands arrive by
 * TMA (4-D tiled maps, OOB zero fill = the conv padding), accumulate in wgmma register fragments (fp32).
 * passes = 3: A_hi.W_hi + A_lo.W_hi + A_hi.W_lo  (fp32-class accuracy, the parity mode)
 * passes = 1: A_hi.W_hi                           (plain bf16)
 * Requirements: Cin % 32 == 0, Cin2 % 32 == 0, Cout % 32 == 0 (K blocks of 64 channels past Cin / Cin2 read TMA
 * zero fill; N tiles past Cout are not stored), taps in {1, 9}, or 4 (2x2 window at rows/cols
 * window_origin..window_origin+1 -- the stride-2 conv on a space-to-depth operand, bbdm_s2d_split; with upsample2x the
 * 4 taps are per output phase), W >= 4.  weights_per_image needs Cin % 64 == 0 and Cout % 64 == 0.
 * Replaces nn.Conv2d 3x3 / 1x1 in ResBlock (openaimodel.py:207,233,244), the qkv / proj_out
 * nn.Conv1d of AttentionBlock (:307,315) and the residual adds (:278,327). */
typedef struct {
  int B, H, W;
  int Cin, Cout, taps;
  const void* a_hi; const void* a_lo;
  const void* w_hi; const void* w_lo;
  const float* bias;
  int Cin2;
  const void* a2_hi; const void* a2_lo;
  const void* w2_hi; const void* w2_lo;
  const float* bias2;
  const float* residual; int res_mode;
  float* out;                 /* fp32 [B,H,W,Cout] or NULL                   */
  void* out_hi; void* out_lo; /* optional split-bf16 copy of the result      */
  int passes;
  int out_nchw_channels;      /* > 0: `out` is NCHW [B, out_nchw_channels, H, W] and only the first
                                 out_nchw_channels (<= Cout) couts are stored (UNet head, replaces
                                 the final layout change); 0: NHWC [B,H,W,Cout]             */
  int upsample2x;             /* 1: the conv input is the nearest-2x upsampling of A (openaimodel.py:118,
                                 212-214) WITHOUT materialising it: A is the low-res tensor [B,H,W,Cin],
                                 the output is [B,2H,2W,Cout]; each output phase (y%2, x%2) is a 2x2
                                 conv whose taps are sums of the 3x3 taps (w_hi/w_lo: [16][Cout][Cin],
                                 index phase*4 + r*2 + c; taps = 4) -- 2.25x fewer MACs than the 3x3
                                 on the upsampled tensor.  residual/res_mode address the OUTPUT grid;
                                 stats_partial then has 4x the rows.                               */
  float* stats_partial;       /* optional: GroupNorm partial sums of the RESULT, fused in the epilogue.
                                 [B * rows_per_image][Cout][2] fp32 (sum, sum of squares), one row per
                                 (128-pixel tile, 32-row warp slice); rows_per_image from
                                 bbdm_conv_umma_geometry.  Ignored (must be NULL) when a tile spans
                                 several images (tiles_per_image == 0).                         */
  int weights_per_image;      /* 1 (taps must be 1): w_hi/w_lo hold one [Cout][Cin] matrix PER IMAGE, [B][Cout][Cin],
                                 and image b is multiplied by matrix b -- B independent GEMMs in one launch (the 36
                                 transform positions of the Winograd path, bbdm_wino_*).  Needs H*W >= 128.  */
  int operand_f16;            /* 1: every operand plane is IEEE fp16 (hi = fp16(x), lo = fp16(x - hi)) instead of
                                 bf16 -- 22 instead of 16 mantissa bits, values must stay below 65504        */
  int window_origin;          /* taps == 4 without upsample2x: first row / column of the 2x2 window.  0: rows/cols 0..1,
                                 zero fill at the bottom/right (the VQGAN Downsample's (0,1,0,1) padding, and the data
                                 gradient of the UNet's stride-2 conv); -1: rows/cols -1..0, zero fill at the top/left
                                 (the UNet Downsample, 3x3 stride 2 padding 1, openaimodel.py:137-163, on the
                                 space-to-depth operand).  Must be 0 otherwise.                                    */
} BbdmConvArgs;
int bbdm_conv_umma(const BbdmConvArgs* a, void* stream);

/* Tile geometry the tensor-core conv uses for an [*,H,W,*] output: pixel box TW x TH x TB (=128)
 * and rows_per_image = 4 * tiles per image of the stats_partial buffer (0 if TB > 1). */
int bbdm_conv_umma_geometry(int H, int W, int* TW, int* TH, int* TB, int* rows_per_image);

/* mean/rstd [B,groups] of cat(t1, t2) from the per-channel partial sums the conv epilogues
 * wrote (part2 may be NULL).  fp64 combine in a fixed order (deterministic).  hw = H*W.
 * Replaces the separate statistics pass (bbdm_gn_stats) for conv-produced tensors. */
int bbdm_gn_finalize_partials(const float* part1, int c1, int rows1, const float* part2, int c2,
                              int rows2, int B, int hw, int groups, float eps, float* mean,
                              float* rstd, void* stream);

/* ------------------------------------------------------------------------------------------
 * Winograd F(4x4, 3x3) path for the stride-1 3x3 ResBlock convolutions (openaimodel.py:207,233): 4x fewer
 * tensor-core MACs.  conv = wino_input -> bbdm_conv_umma(weights_per_image, operand_f16; B = 36 positions,
 * H = tiles/16, W = 16, taps = 1, out = M) -> wino_output.  Split-FP16 operands carry 22 mantissa bits; the
 * deviation of the chain from the fp64 conv is set by the position GEMMs' accumulation, which the output transform
 * amplifies: on an H100 80GB HBM3 (400 W) 5.6e-6 to 9.6e-6 at every weight std from 2e-2 to 1e-4, against 4.5e-6
 * for the direct split-bf16 kernel (tests/test_gpu_winograd_range.py).  Promoting every K-block
 * (BBDM_WINO_CHUNK=1) brings it to the direct kernel's level.
 * ------------------------------------------------------------------------------------------ */

/* tiles_h = H/4, tiles_w = W/4, tiles_total = B*tiles_h*tiles_w; eligible = 1 iff H, W are multiples of 4 and
 * tiles_total is a multiple of 16 and >= 128 (the GEMM's M blocking). */
int bbdm_wino_geometry(int B, int H, int W, int* tiles_h, int* tiles_w, int64_t* tiles_total, int* eligible);

/* cat(src1, src2) [B,H,W,C] fp32 -> act = silu?(GN_affine(x) * (1+film_scale) + film_shift) (as bbdm_prep_operand)
 * -> V = B^T act B for every 6x6 tile (stride 4, origin (-1,-1), zero padding of the ACTIVATED tensor) ->
 * split-fp16 planes v_hi, v_lo [36][tiles_total][C].  raw_hi/raw_lo (optional): split-bf16 NHWC planes of the
 * raw input (A operand of the ResBlock's 1x1 skip convolution, openaimodel.py:244).
 * mean == NULL (silu must be 0): identity -- the tensor is transformed as it is (the data-gradient convolution of
 * the training path transforms dY).
 * Range: V is stored as fp16 (largest finite 65504) and B^T d B amplifies a tile by at most 100, so max|act| <= 655
 * is finite for every input; on GroupNorm-normalised random inputs the first non-finite result came at
 * max|act| ~ 4100 (2060 was finite; tools/wino_activation_window.py, H100).  The forward route does not guard
 * against larger activations: they give inf/NaN. */
typedef struct {
  const float* src1; int c1;
  const float* src2; int c2;
  int B, H, W;
  int groups;
  const float* mean; const float* rstd; const float* gamma; const float* beta;
  const float* film_scale; const float* film_shift; int64_t film_stride;
  int silu;
  void* v_hi; void* v_lo;
  void* raw_hi; void* raw_lo;
  void* act_hi; void* act_lo;   /* optional: split-bf16 NHWC planes of the ACTIVATED tensor (training: operand of the
                                   weight-gradient GEMM, bbdm_conv_wgrad) */
  int down2;                    /* F(6,3) only: see bbdm_wino6_input below */
} BbdmWinoInputArgs;
int bbdm_wino_input(const BbdmWinoInputArgs* a, void* stream);

/* m [36][tiles_total][Cout] fp32 (the position GEMMs' output) -> out [B,H,W,Cout] = inv_wscale * A^T m A + bias
 * (+ residual, addressed as in BbdmConvArgs.res_mode), and optionally the GroupNorm partial sums of the result:
 * stats_partial [B * tiles_h][Cout][2] (rows_per_image = tiles_h for bbdm_gn_finalize_partials). */
typedef struct {
  const float* m;
  const float* inv_wscale;   /* device float 1/s written by bbdm_wino_pack_weight for the weight planes; NULL: the
                                fixed 2^-8 of planes packed without a scale buffer */
  int B, H, W, Cout;
  const float* bias;
  const float* residual; int res_mode;
  float* out;
  float* stats_partial;
  int up2_phases;            /* F(6,3) only, res_mode 0: see bbdm_wino6_output below */
} BbdmWinoOutputArgs;
int bbdm_wino_output(const BbdmWinoOutputArgs* a, void* stream);

/* w [Cout,Cin,3,3] fp32 -> U = s * G w G^T (fp64 arithmetic), split-fp16 planes u_hi, u_lo [36][Cout][Cin], with
 * the per-tensor power of two s = 2^(14 - ceil(log2 max|w|)) (2^8 for an all-zero tensor), so that |U| <= 2^14 and
 * the planes stay normal fp16 numbers at any weight magnitude.  max|w| is reduced on the device (deterministic) and
 * 1/s is written to the device float *inv_wscale, which bbdm_wino_output takes: no host synchronisation, and a
 * stable address for graph replay.  inv_wscale == NULL: the fixed s = 2^8 (exact for N(0, 0.02)-scale weights; the
 * lo planes of much smaller weights become fp16 subnormals).  dgrad != 0: the planes of the data-gradient convolution instead
 * ([36][Cin][Cout], kernel flipped, channels swapped; cf. bbdm_pack_weight_split_dgrad). */
int bbdm_wino_pack_weight(const float* w, int Cout, int Cin, int dgrad, void* u_hi, void* u_lo, float* inv_wscale,
                          void* stream);

/* Winograd F(6x6, 3x3) forms of the four calls above (interpolation points 0, +-1, +-2, +-1/2): 64 transform
 * positions per 6x6 output tile, 0.79x the position-GEMM MACs of F(4,3) per output pixel, for the large maps.
 * The arguments are the same; what differs:
 *   geometry     tiles_h = ceil(H/6), tiles_w = ceil(W/6) (any H, W: edge tiles read the zero padding of the
 *                activated tensor and store nothing past H or W); tiles_total = B*tiles_h*tiles_w rounded up to a
 *                multiple of 16 and to at least 128 -- the rows of V and M, the GEMM's H = tiles_total/16
 *                (wino6_input writes the padding rows as zeros); eligible = 1 for every shape.
 *   input        v_hi, v_lo [64][tiles_total][C]; c1 and c2 must be multiples of 64.  Range: B^T d B amplifies a
 *                tile by at most 225 (F(4,3): 100), so max|act| <= 291 is finite for every input; a V value
 *                that is not a finite fp16 number sets the device fault word to 0xC0000000 | C
 *                (bbdm_check_device_fault reports it).
 *                down2 != 0: the conv's input is the 2x2 average pool of the activated [B,H,W,C] sources (the
 *                down-ResBlock's in_layers -> h_upd order: activate every pixel, then average), so the transform
 *                and the geometry are those of the H/2 x W/2 map; no raw or act planes.
 *   output      m [64][tiles_total][Cout]; stats_partial [B * tiles_h][Cout][2].
 *                up2_phases != 0: the output of a nearest-2x upsample followed by a 3x3 conv, run as one 3x3 conv on
 *                the H x W (low-res) map with 4*Cout outputs, phase-major: channel phase*Cout + co of m is output
 *                channel co at the pixels (2y+a, 2x+b) of out [B, 2H, 2W, Cout], phase = 2a + b.  bias [Cout];
 *                no residual; stats_partial [B * tiles_h * 4][Cout][2] (rows_per_image = 4 * tiles_h).
 *   pack_weight  u_hi, u_lo [64][Cout][Cin] (dgrad: [64][Cin][Cout]); the same scale s (|s U| <= 1.55 * 2^14). */
int bbdm_wino6_geometry(int B, int H, int W, int* tiles_h, int* tiles_w, int64_t* tiles_total, int* eligible);
int bbdm_wino6_input(const BbdmWinoInputArgs* a, void* stream);
int bbdm_wino6_output(const BbdmWinoOutputArgs* a, void* stream);
int bbdm_wino6_pack_weight(const float* w, int Cout, int Cin, int dgrad, void* u_hi, void* u_lo, float* inv_wscale,
                           void* stream);

/* General fp32 direct convolution on CUDA cores (any Cin/Cout, k in {1,3}, stride 1 or 2,
 * pad k/2): stem (openaimodel.py:524), head (:690), conv-mode Downsample/Upsample (:109,150)
 * and channel counts the tensor-core kernel does not take.  src NHWC fp32 [B,H,W,Cin],
 * w_packed from bbdm_pack_weight_f32, out [B,Ho,Wo,Cout]; residual [B,Ho,Wo,Cout] or NULL. */
int bbdm_conv_direct(const float* src, const float* w_packed, const float* bias,
                     const float* residual, float* out, int B, int H, int W, int Cin, int Cout,
                     int k, int stride, void* stream);

/* UNet stem (openaimodel.py:524, Conv2d(in_channels, model_channels, 3, padding=1) with 3..16 input channels) as a
 * dedicated kernel: weights resident in shared memory, one CTA per image row, and the GroupNorm partial sums of the
 * output fused in (stats_partial [B*H][Cout][2], rows_per_image = H; may be NULL).  Same fp32 FMA order as
 * bbdm_conv_direct => identical bits.  Needs W %% 32 == 0, Cin <= 16, Cout in {32, 64, 96, 128}. */
int bbdm_conv_stem(const float* src, const float* w_packed, const float* bias, float* out, int B, int H, int W,
                   int Cin, int Cout, float* stats_partial, void* stream);

/* The same kernel with explicit zero padding (pad_lo before, pad_hi after, each < k): the VQGAN
 * Downsample pads (0,1,0,1) and strides by 2 (model/VQGAN/model.py:55-73).
 * out [B,Ho,Wo,Cout] with Ho = (H + pad_lo + pad_hi - k)/stride + 1. */
int bbdm_conv_direct_pad(const float* src, const float* w_packed, const float* bias,
                         const float* residual, float* out, int B, int H, int W, int Cin, int Cout,
                         int k, int stride, int pad_lo, int pad_hi, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training: gradients of the tensor-core convolution
 *   data gradient   dX = conv(dY, W^T flipped)  -> bbdm_conv_umma with re-packed weights
 *   weight gradient dW                          -> bbdm_conv_wgrad (below)
 * Replaces the autograd of nn.Conv2d in ResBlock (openaimodel.py:207,233,244) during
 * loss.backward() (runners/BaseRunner.py:412).
 * ------------------------------------------------------------------------------------------ */

/* fp32 NHWC gradient src [P][C] (P = B*H*W) -> split-bf16 planes in both orientations
 *   hi/lo     [P][C]  (may be NULL)  : A operand of the data-gradient conv
 *   hi_t/lo_t [C][P], rows ld_t >= P elements apart : A operand (K = pixels) of the weight-gradient GEMM
 *                                    (which needs ld_t % 8 == 0: allocate P rounded up to 8)
 * and, if colsum != NULL, colsum[c] = sum_p src[p][c] (the bias gradient; deterministic).
 * workspace: ceil(P/64)*C floats (only needed with colsum). */
int bbdm_split_grad(const float* src, int64_t P, int C, void* hi, void* lo, void* hi_t, void* lo_t, int64_t ld_t,
                    float* colsum, float* workspace, void* stream);

/* split-K factor and workspace size (floats) bbdm_conv_wgrad needs for this problem (Cin, Cout % 32 == 0). */
int bbdm_conv_wgrad_workspace(int B, int H, int W, int Cin, int Cout, int taps, int* splits,
                              int64_t* floats);

/* dW[co][ci][ky][kx] (OIHW fp32, overwritten) = sum_p dY[p][co] * A[p + tap][ci] on wgmma:
 * g_hi_t/g_lo_t = dY^T planes [Cout][P] from bbdm_split_grad, rows ld_g elements apart (ld_g >= P, a multiple of 8),
 * a_hi/a_lo = the forward conv's operand planes [B,H,W,Cin].  M = Cout, N = Cin, K = pixels in blocks of 64 consecutive
 * pixels of the flattened (b, h, w) index (any map size and batch; the last block is zero-filled past P); split-bf16
 * x3; split-K partials reduced in a fixed order.  Requirements: Cin, Cout % 32 == 0, W >= 4, taps in {1, 9}
 * (window_origin 0), or 4 (2x2 window at rows/cols window_origin..window_origin+1, window_origin 0 or -1, as in
 * BbdmConvArgs; dw is then [Cout][Cin][2][2]). */
int bbdm_conv_wgrad(const void* g_hi_t, const void* g_lo_t, int64_t ld_g, const void* a_hi, const void* a_lo,
                    int B, int H, int W, int Cin, int Cout, int taps, int window_origin, float* dw,
                    float* workspace, void* stream);

/* Weight gradient of the small-channel fp32 convolutions (UNet stem / head, the SpatialTransformer's k|v
 * projection of the few-channel context; Cin*Cout <= 2^24):
 * dy NHWC [B,H,W,Cout], x NHWC [B,H,W,Cin] fp32, stride 1, pad k/2 -> dw OIHW fp32 (overwritten).
 * workspace: any multiple of k*k*Cin*Cout floats (more = more CTAs, up to 4096); fixed-order reduce.
 * (The data gradient of these layers is bbdm_conv_direct with the flipped/transposed weights.) */
int bbdm_conv_wgrad_direct(const float* dy, const float* x, int B, int H, int W, int Cin, int Cout, int k,
                           float* dw, float* workspace, int64_t workspace_floats, void* stream);

/* Backward of the fused operand preparation  a = silu( (gamma*xh + beta) * (1+scale) + shift ),
 * xh = (x-mean)*rstd  (training path; replaces the autograd of GroupNorm32 + SiLU + scale-shift,
 * openaimodel.py:205-206,229-230,270-274).  Two HBM-bound passes over (x, dA):
 *   bbdm_gn_bwd_reduce : a12[b][c] = (sum_p dz, sum_p dz*xh), dz = dA*silu'(z); workspace B*64*C*2 floats
 *   bbdm_gn_bwd_apply  : dx = rstd*(dz*gamma*(1+scale) - (s1 + xh*s2)/n) with the per-(b,group) sums
 *                        s1, s2 the host derives from a12 (as are dgamma, dbeta, dscale, dshift). */
int bbdm_gn_bwd_reduce(const float* x, const float* da, int B, int H, int W, int C, int groups,
                       const float* mean, const float* rstd, const float* gamma, const float* beta,
                       const float* film_scale, const float* film_shift, int64_t film_stride, int silu,
                       float* a12, float* workspace, void* stream);
int bbdm_gn_bwd_apply(const float* x, const float* da, int B, int H, int W, int C, int groups,
                      const float* mean, const float* rstd, const float* gamma, const float* beta,
                      const float* film_scale, const float* film_shift, int64_t film_stride, int silu,
                      const float* s1, const float* s2, float* dx, void* stream);

/* ------------------------------------------------------------------------------------------
 * SpatialTransformer pieces (reference base/modules/attention.py:36-264).  The 1x1 projections
 * and every nn.Linear run on bbdm_conv_umma (taps = 1 over the [B, H, W, C] token grid); these are the remaining ops.
 * ------------------------------------------------------------------------------------------ */

/* nn.LayerNorm(C) over the last dimension of x [rows][C] (biased variance, eps inside the sqrt, affine), fp32
 * and/or split-bf16 output (operand of the following Linear).  Replaces norm1/2/3 of BasicTransformerBlock
 * (attention.py:203-205, 213-215).  C even, <= 2048. */
int bbdm_layernorm_split(const float* x, int64_t rows, int C, const float* gamma, const float* beta, float eps,
                         float* out_f32, void* out_hi, void* out_lo, void* stream);

/* GEGLU gate (attention.py:36-43): u [rows][2N] = the projection's output -> out[r][n] = u[r][n] * gelu(u[r][N+n])
 * (exact erf GELU), fp32 and/or split-bf16. */
int bbdm_geglu_split(const float* u, int64_t rows, int N, float* out_f32, void* out_hi, void* out_lo, void* stream);

/* Cross-attention core (CrossAttention.forward, attention.py:166-192): queries q [B,Tq,C] and keys|values
 * kv [B,Tkv,2C] (k = columns [0,C), v = [C,2C)), both as split-bf16 planes, head h = columns h*D..(h+1)*D of each;
 * out[b,i,:] = softmax_j(q_i.k_j * D^-1/2) v_j per head, flash-style (no Tq x Tkv buffer).  D: a multiple of 8 up to 256. */
int bbdm_attention_cross(const void* q_hi, const void* q_lo, const void* kv_hi, const void* kv_lo, int B, int Tq,
                         int Tkv, int C, int heads, float* out_f32, void* out_hi, void* out_lo, void* stream);

/* Training backward of the three ops above.
 * bbdm_layernorm_bwd: x [rows][C] (the forward's input; mean / rstd are recomputed), dy [rows][C] -> dx [rows][C],
 *   dgamma / dbeta [C] (fixed-order column sums, deterministic).  workspace: ceil(rows/64) * 2C floats.  C even, <= 2048.
 * bbdm_geglu_bwd: u [rows][2N] (the forward's input), dy [rows][N] -> du [rows][2N] = [dy*gelu(g) | dy*a*gelu'(g)].
 * bbdm_attention_cross_bwd: fp32 q [B,Tq,C], kv [B,Tkv,2C] and out [B,Tq,C] of bbdm_attention_cross, dout [B,Tq,C] ->
 *   dq [B,Tq,C], dkv [B,Tkv,2C]; the probabilities are recomputed tile by tile (no Tq x Tkv buffer), exact fp32.
 *   lse / delta: [B*heads*Tq] fp32 workspaces.  D: a multiple of 8 up to 256; the same kernels as bbdm_attention_bwd. */
int bbdm_layernorm_bwd(const float* x, const float* dy, int64_t rows, int C, const float* gamma, float eps, float* dx,
                       float* dgamma, float* dbeta, float* workspace, void* stream);
int bbdm_geglu_bwd(const float* u, const float* dy, int64_t rows, int N, float* du, void* stream);
int bbdm_attention_cross_bwd(const float* q, const float* kv, const float* out, const float* dout, int B, int Tq, int Tkv,
                             int C, int heads, float* dq, float* dkv, float* lse, float* delta, void* stream);

/* SpatialRescaler, the latent model's cond-stage encoder (model/BrownianBridge/base/modules/encoders/modules.py:106-134:
 * n_stages x F.interpolate(scale_factor=0.5, mode='bilinear') then an optional 1x1 Conv2d channel_mapper), no-grad path,
 * one launch.  src [B,C,H,W] fp32 (C <= 16); w [Cout,C] / bias [Cout] or NULL (no channel map: Cout ignored);
 * out [B, Cout or C, H >> n_stages, W >> n_stages] fp32 NCHW -- the `context` the UNet stem concatenates
 * (openaimodel.py:741-744).  0 <= n_stages <= 4.  Each stage is the exact 2x2 expression of the bilinear kernel at
 * scale 0.5 (both weights 0.5). */
int bbdm_spatial_rescale(const float* src, int B, int C, int H, int W, int n_stages, const float* w, const float* bias,
                         int Cout, float* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Output path of sample_to_eval
 * ------------------------------------------------------------------------------------------ */

/* images [B,C,H,W] fp32 -> out [B,H,W,C] uint8: clamp(x*0.5+0.5, 0, 1) (if to_normal), then
 * clamp(x*255+0.5, 0, 255) truncated to uint8 -- the per-image expression of save_single_image
 * (runners/utils.py:67-74: mul_(0.5).add_(0.5).clamp_(0,1).mul_(255).add_(0.5).clamp_(0,255).permute(1,2,0)
 * .to(uint8)), same operation order => byte-exact, for the whole batch in one launch. */
int bbdm_denorm_to_uint8(const float* images, int B, int C, int H, int W, int to_normal, uint8_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-tensor optimizer / EMA updates: one launch over every parameter tensor.
 * params/grads: DEVICE arrays of n tensor pointers (fp32; a NULL gradient skips that tensor like torch does);
 * numel/state_off: DEVICE int64 [n] (elements, offset of the tensor's state inside the flat exp_avg / exp_avg_sq /
 * shadow buffers); chunk_tensor/chunk_index: DEVICE int32 [n_chunks], one entry per CTA = (tensor, chunk of
 * bbdm_optim_chunk_elems() elements).
 * ------------------------------------------------------------------------------------------ */
int bbdm_optim_chunk_elems(void);

/* torch.optim.Adam's update (the optimizer runners/utils.py:48-57 builds, stepped at runners/BaseRunner.py:413),
 * non-amsgrad, L2 weight decay, `step` = the 1-based step count of this update.  The hyper-parameters are doubles like
 * the python floats torch.optim.Adam holds: 1 - beta1, 1 - beta2 and the bias corrections are computed from them in
 * fp64, as torch does, before each is rounded to fp32 once.  ema_shadow != NULL additionally applies shadow = (1-ema_decay)*p_new + ema_decay*shadow in the same
 * pass (runners/base/EMA.py:21-29 with with_decay=True). */
int bbdm_adam_multi(void* const* params, const void* const* grads, const int64_t* numel, const int64_t* state_off,
                    const int32_t* chunk_tensor, const int32_t* chunk_index, int n_chunks, float* exp_avg,
                    float* exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay, int64_t step,
                    float* ema_shadow, double ema_decay, void* stream);

/* The same update in the capturable form of torch.optim.Adam(capturable=True): the step count and the learning rate
 * live in DEVICE memory, so a CUDA graph that captures this call replays it with the count advancing and the rate its
 * owner last wrote.  `step` (fp32 scalar) is incremented on the device first, then the update reads it (the 1-based
 * count of this update); `lr` is an fp64 scalar.  The bias corrections are formed in the kernel from those values with
 * the expressions of bbdm_adam_multi, in fp64, so an eager sequence of calls matches bbdm_adam_multi with the same
 * counts.  ema_shadow / ema_decay as in bbdm_adam_multi.  Two launches (increment, update). */
int bbdm_adam_multi_dev(void* const* params, const void* const* grads, const int64_t* numel, const int64_t* state_off,
                        const int32_t* chunk_tensor, const int32_t* chunk_index, int n_chunks, float* exp_avg,
                        float* exp_avg_sq, float* step, const double* lr, double beta1, double beta2, double eps,
                        double weight_decay, float* ema_shadow, double ema_decay, void* stream);

/* EMA.update (runners/base/EMA.py:21-29): shadow = (1-decay)*param + decay*shadow (the reference's operation
 * order with the python-float scalars (1.0 - decay) and decay each rounded to fp32: bit-exact), or shadow = param
 * when with_decay == 0.  decay is a double like the python attribute. */
int bbdm_ema_multi(const void* const* params, const int64_t* numel, const int64_t* state_off,
                   const int32_t* chunk_tensor, const int32_t* chunk_index, int n_chunks, float* shadow, double decay,
                   int with_decay, void* stream);

/* ------------------------------------------------------------------------------------------
 * Attention core
 * ------------------------------------------------------------------------------------------ */

/* softmax((q*s)(k*s)^T) v per head, s = head_dim^-1/4, fp32 softmax, flash-style (no T x T
 * buffer).  qkv: fp32 [B,T,3C] in the channel order of the reference's qkv conv:
 *   order 0 (QKVAttentionLegacy, openaimodel.py:350-375): [head][q|k|v][head_dim]
 *   order 1 (QKVAttention, :382-413):                      [q|k|v][head][head_dim]
 * out: fp32 [B,T,C] and/or split bf16 (A operand of the proj_out GEMM).
 * Split-bf16 tensor-core products with fp32 accumulation: q and k are scaled by s, then split; expf softmax.
 * Runs on the mma.sync kernel of bbdm_attention_split, which copies the fp32 K/V tiles with cp.async and splits
 * them in shared memory.  head_dim: a multiple of 8 up to 256. */
int bbdm_attention(const float* qkv, int B, int T, int C, int heads, int order,
                   float* out_f32, void* out_hi, void* out_lo, void* stream);

/* Same attention core on PRE-SPLIT bf16 planes qkv_hi/qkv_lo [B,T,3C] (written by the qkv
 * conv's epilogue, BbdmConvArgs.out_hi/out_lo): no conversion or re-splitting of K/V per query
 * tile; cp.async double-buffered KV tiles, ldmatrix fragments, 128 queries per CTA over 64-key tiles (head_dim
 * above 128: 64 queries over 32-key tiles); S is scaled by D^-1/2 after the products and the softmax runs on
 * ex2.approx.  head_dim: a multiple of 8 up to 256. */
int bbdm_attention_split(const void* qkv_hi, const void* qkv_lo, int B, int T, int C, int heads,
                         int order, float* out_f32, void* out_hi, void* out_lo, void* stream);

/* The same computation as a FlashAttention-style WARP-SPECIALISED wgmma kernel (head_dim 64 or 128):
 * TMA-staged Q / K / V tiles, S = Q K^T and O = P V on wgmma with register accumulators (V
 * consumed as an MN-major operand, P fed back from registers as the A operand), two 64-query
 * warpgroups per CTA, fp32 register accumulation of O with the
 * online-softmax rescale.  head_dim in {64,128}; returns BBDM_E_UNSUPPORTED for other head dims. */
int bbdm_attention_tc(const void* qkv_hi, const void* qkv_lo, int B, int T, int C, int heads,
                      int order, float* out_f32, void* out_hi, void* out_lo, void* stream);

/* Backward of the attention core (training; replaces the autograd + checkpoint() recompute of
 * QKVAttentionLegacy / QKVAttention, openaimodel.py:318,350-413, util.py:119-148): given qkv [B,T,3C],
 * out = attention(qkv) [B,T,C] and dout [B,T,C] (all fp32), writes dqkv [B,T,3C].  FlashAttention-style
 * recompute in exact fp32 -- no T x T tensor.  lse, delta: fp32 workspaces of B*heads*T elements each.
 * head_dim: a multiple of 8 up to 256 (above 128 the streamed operands share one shared-memory tile);
 * deterministic. */
int bbdm_attention_bwd(const float* qkv, const float* out, const float* dout, int B, int T, int C, int heads,
                       int order, float* dqkv, float* lse, float* delta, void* stream);

/* Repack of attention heads whose width d is not a multiple of 8, so that the kernels above run them at
 * dp = d rounded up to 8.  A row holds G = tensors * heads groups of d columns (one head's q, k or v): order 0 puts
 * the tensors of a head together (the legacy qkv layout), order 1 all heads of one tensor together (q, k|v, dout).
 * Every value of a group is multiplied by its tensor's scale (scale0..2; the caller folds (dp/d)^(1/4) into q and k,
 * so the kernels' dp^-1/2 softmax scale becomes d^-1/2), with one fp32 rounding.
 *   pad:   src [rows, G*d] fp32 -> [rows, G*dp], zeros in columns d..dp-1 of every group; out_f32 16-byte aligned,
 *          the planes 8-byte aligned.
 *   unpad: src [rows, G*dp] fp32 -> [rows, G*d].
 * out: fp32 and/or split-bf16 planes (hi = bf16(x), lo = bf16(x - hi), as bbdm_prep_operand splits).  tensors 1..3.
 * No host synchronisation or allocation (capturable). */
int bbdm_attention_pad_heads(const float* src, int64_t rows, int heads, int tensors, int d, int order, float scale0,
                             float scale1, float scale2, float* out_f32, void* out_hi, void* out_lo, void* stream);
int bbdm_attention_unpad_heads(const float* src, int64_t rows, int heads, int tensors, int d, int order, float scale0,
                               float scale1, float scale2, float* out_f32, void* out_hi, void* out_lo, void* stream);

/* ---- VQGAN ends of the latent models ---------------------------------------
 * Row softmax of a [rows, cols] fp32 score matrix, p = softmax(scale * s), written as split-bf16 planes
 * (A operand of the P.V GEMM of the single-head AttnBlock, model/VQGAN/model.py:168-183). cols % 4 == 0.
 * Only the first valid_cols (1..cols) columns of a row enter its max and sum; the planes hold exact zeros in
 * the rest (the padding of a token axis rounded up to the GEMM tile).  valid_cols == cols: the whole row. */
int bbdm_softmax_rows_split(const float* src, int64_t rows, int64_t cols, int64_t valid_cols, float scale,
                            void* out_hi, void* out_lo, void* stream);

/* Backward of that row softmax, for attention run as two GEMMs around it (heads wider than the flash kernels take):
 * from the scores s and dp = dL/dp ([rows, cols] fp32, row-major), recomputes p = softmax(scale * s) over the first
 * valid_cols columns with bbdm_softmax_rows_split's max, sum and expf order, and writes the score gradient
 * ds = scale * p * (dp - sum_j p_j dp_j) as split-bf16 planes (exact zeros past valid_cols).  cols % 4 == 0.
 * Deterministic (fixed reduction order). */
int bbdm_softmax_rows_bwd(const float* s, const float* dp, int64_t rows, int64_t cols, int64_t valid_cols, float scale,
                          void* ds_hi, void* ds_lo, void* stream);

/* Space-to-depth by 2 with bf16 split: src [B,H,W,C] fp32 -> planes [B,H/2,W/2,4C], channel
 * (row parity*2 + col parity)*C + c.  With it the VQGAN Downsample (zero-pad (0,1,0,1) + 3x3 stride-2 conv,
 * model/VQGAN/model.py:55-73) runs on the tensor cores as a 2x2-tap convolution over 4C channels
 * (BbdmConvArgs.taps = 4: window rows/cols (0..1), zero padding at the bottom/right). H, W even; C % 4 == 0. */
int bbdm_s2d_split(const float* src, int B, int H, int W, int C, void* out_hi, void* out_lo, void* stream);

/* VectorQuantizer2.forward (model/VQGAN/quantize.py:271-312): for every latent vector z [n_vectors, dim]
 * (NHWC order) the index of the nearest codebook row, d = (|z|^2 + |e|^2) - 2 z.e in fp32, first minimum;
 * z_q = z + (e - z) (forward value of the straight-through expression).  dim <= 16. */
int bbdm_vq_nearest(const float* z, const float* codebook, int64_t n_vectors, int n_embed, int dim,
                    float* z_q, long long* indices, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BBDM_B200_H_ */
