// Host-side check of the phase-stacked nearest-2x form of the Winograd F(6x6,3x3) output transform
// (bbdm_b200/csrc/winograd.cu, wino6_output_tile<WINO6_UP_PHASES>, a __host__ __device__ function): the SAME source the
// kernel runs is executed on the CPU for every (sample, tile, channel), edge tiles past h or w included, and compared
// with a direct fp64 evaluation of out = inv_wscale * A^T M A + bias at the interleaved output pixels, plus the
// per-thread partial sums that feed the fused GroupNorm statistics.  No GPU and no CUDA runtime call is involved.
// Build + run (tests/test_wino6_up2_output_host.py does this):
//     nvcc -std=c++17 --expt-relaxed-constexpr -I include -o /tmp/host_check_wino6_up2_output tools/host_check_wino6_up2_output.cu
#include "../bbdm_b200/csrc/winograd.cu"

#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

static const double AT[6][8] = {{1, 1, 1, 1, 1, 1, 1, 0},
                                {0, 1, -1, 2, -2, 0.5, -0.5, 0},
                                {0, 1, 1, 4, 4, 0.25, 0.25, 0},
                                {0, 1, -1, 8, -8, 0.125, -0.125, 0},
                                {0, 1, 1, 16, 16, 0.0625, 0.0625, 0},
                                {0, 1, -1, 32, -32, 0.03125, -0.03125, 1}};

// The phase-stacked nearest-2x form (WINO6_UP_PHASES): M has 4*Cout channels phase*Cout + co on the h x w tile grid;
// output pixel (2y+a, 2x+b), channel co, of the [B, 2h, 2w, Cout] result is pixel (y, x) of channel (2a+b)*Cout + co.
static int run_up(int B, int h, int w, int Cout, bool with_bias, float inv) {
  using namespace bbdm;
  std::mt19937 rng(4321 + h * 31 + w);
  std::normal_distribution<float> nd(0.f, 1.f);
  const int th = (h + 5) / 6, tw = (w + 5) / 6, C4 = 4 * Cout, H = 2 * h, W = 2 * w;
  const int64_t Mtot = ((int64_t)B * th * tw + 15) / 16 * 16;
  std::vector<float> M((size_t)64 * Mtot * C4), bias(Cout), out((size_t)B * H * W * Cout, -777.f);
  for (auto& v : M) v = 40.f * nd(rng);
  for (auto& v : bias) v = nd(rng);
  WinoOutParams p;
  p.m = M.data(); p.Mtot = Mtot; p.B = B; p.H = h; p.W = w; p.Cout = Cout; p.th = th; p.tw = tw;
  p.bias = with_bias ? bias.data() : nullptr;
  p.residual = nullptr; p.res_mode = BBDM_RES_NONE;
  p.out = out.data(); p.stats = nullptr;
  std::vector<double> s1((size_t)Cout, 0.0), s2((size_t)Cout, 0.0);
  for (int b = 0; b < B; ++b)
    for (int ty = 0; ty < th; ++ty)
      for (int tx = 0; tx < tw; ++tx)
        for (int c = 0; c < C4; ++c) {
          float a0 = 0, q0 = 0;
          wino6_output_tile<WINO6_UP_PHASES>(p, b, ty, tx, c, with_bias ? bias[c % Cout] : 0.f, inv, a0, q0);
          s1[c % Cout] += a0; s2[c % Cout] += q0;
        }
  double worst = 0, scale = 0, r1 = 0, r2 = 0;
  std::vector<double> w1((size_t)Cout, 0.0), w2((size_t)Cout, 0.0);
  for (int b = 0; b < B; ++b)
    for (int hh = 0; hh < H; ++hh)
      for (int ww = 0; ww < W; ++ww)
        for (int co = 0; co < Cout; ++co) {
          const int y = hh / 2, x = ww / 2, c = ((hh & 1) * 2 + (ww & 1)) * Cout + co;
          const int ty = y / 6, i = y % 6, tx = x / 6, j = x % 6;
          const int64_t m = ((int64_t)b * th + ty) * tw + tx;
          double v = 0;
          for (int k = 0; k < 8; ++k)
            for (int l = 0; l < 8; ++l) v += AT[i][k] * (double)M[((size_t)(k * 8 + l) * Mtot + m) * C4 + c] * AT[j][l];
          v = v * (double)inv + (with_bias ? (double)bias[co] : 0.0);
          const double got = out[(((size_t)b * H + hh) * W + ww) * Cout + co];
          worst = std::fmax(worst, std::fabs(got - v));
          scale = std::fmax(scale, std::fabs(v));
          w1[co] += got; w2[co] += got * got;
        }
  for (int c = 0; c < Cout; ++c) {
    r1 = std::fmax(r1, std::fabs(s1[c] - w1[c]) / (1.0 + std::fabs(w1[c])));
    r2 = std::fmax(r2, std::fabs(s2[c] - w2[c]) / (1.0 + std::fabs(w2[c])));
  }
  const bool ok = worst <= 2e-6 * scale && r1 < 1e-4 && r2 < 1e-4;
  std::printf("UP2_PHASES B=%d h=%d w=%d Cout=%d bias=%d 1/s=%g: max abs dev %.3e (scale %.3e), partial sums %.1e / %.1e -> %s\n",
              B, h, w, Cout, (int)with_bias, inv, worst, scale, r1, r2, ok ? "ok" : "FAIL");
  return ok ? 0 : 1;
}

int main() {
  int bad = 0;
  // ragged low-res maps (h or w not multiples of 6) exercise the masked edge tiles
  bad += run_up(2, 13, 10, 64, true, 1.0f / 4096);
  bad += run_up(1, 12, 6, 128, false, 1.0f / 256);
  bad += run_up(1, 7, 19, 192, true, 1.0f / 131072);
  std::printf(bad ? "FAILED\n" : "ALL OK\n");
  return bad;
}
