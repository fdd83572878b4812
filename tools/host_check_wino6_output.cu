// Host-side check of the Winograd F(6x6,3x3) output transform's tile routine (bbdm_b200/csrc/winograd.cu,
// wino6_output_tile<RES>, a __host__ __device__ function): the SAME source the kernel runs is executed on the CPU for
// every (sample, tile, channel), edge tiles past H or W included, and compared with a direct fp64 evaluation of
//     out = inv_wscale * A^T M A + bias + residual(same | nearest-up | 2x2-average addressed)
// plus the per-thread partial sums that feed the fused GroupNorm statistics.  No GPU and no CUDA runtime call is
// involved.  Build + run (tests/test_wino6_output_host.py does this):
//     nvcc -std=c++17 --expt-relaxed-constexpr -I include -o /tmp/host_check_wino6_output tools/host_check_wino6_output.cu
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

template <int RES>
static int run(int B, int H, int W, int Cout, bool with_bias, float inv) {
  using namespace bbdm;
  std::mt19937 rng(1234 + RES * 7 + H);
  std::normal_distribution<float> nd(0.f, 1.f);
  const int th = (H + 5) / 6, tw = (W + 5) / 6;
  const int64_t Mtot = ((int64_t)B * th * tw + 15) / 16 * 16;
  std::vector<float> M((size_t)64 * Mtot * Cout), bias(Cout), out((size_t)B * H * W * Cout, -777.f);
  for (auto& v : M) v = 40.f * nd(rng);
  for (auto& v : bias) v = nd(rng);
  int RH = H, RW = W;
  if (RES == BBDM_RES_UP2) { RH = H / 2; RW = W / 2; }
  if (RES == BBDM_RES_DOWN2) { RH = H * 2; RW = W * 2; }
  std::vector<float> res((size_t)B * RH * RW * Cout);
  for (auto& v : res) v = nd(rng);
  WinoOutParams p;
  p.m = M.data(); p.Mtot = Mtot; p.B = B; p.H = H; p.W = W; p.Cout = Cout; p.th = th; p.tw = tw;
  p.bias = with_bias ? bias.data() : nullptr;
  p.residual = RES == BBDM_RES_NONE ? nullptr : res.data(); p.res_mode = RES;
  p.out = out.data(); p.stats = nullptr;
  std::vector<double> s1((size_t)Cout, 0.0), s2((size_t)Cout, 0.0);
  for (int b = 0; b < B; ++b)
    for (int ty = 0; ty < th; ++ty)
      for (int tx = 0; tx < tw; ++tx)
        for (int c = 0; c < Cout; ++c) {
          float a0 = 0, q0 = 0;
          wino6_output_tile<RES>(p, b, ty, tx, c, with_bias ? bias[c] : 0.f, inv, a0, q0);
          s1[c] += a0; s2[c] += q0;
        }
  double worst = 0, scale = 0, r1 = 0, r2 = 0;
  std::vector<double> w1((size_t)Cout, 0.0), w2((size_t)Cout, 0.0);
  for (int b = 0; b < B; ++b)
    for (int hh = 0; hh < H; ++hh)
      for (int ww = 0; ww < W; ++ww)
        for (int c = 0; c < Cout; ++c) {
          const int ty = hh / 6, i = hh % 6, tx = ww / 6, j = ww % 6;
          const int64_t m = ((int64_t)b * th + ty) * tw + tx;
          double y = 0;
          for (int k = 0; k < 8; ++k)
            for (int l = 0; l < 8; ++l) y += AT[i][k] * (double)M[((size_t)(k * 8 + l) * Mtot + m) * Cout + c] * AT[j][l];
          y = y * (double)inv + (with_bias ? (double)bias[c] : 0.0);
          if (RES == BBDM_RES_SAME) y += res[(((size_t)b * H + hh) * W + ww) * Cout + c];
          if (RES == BBDM_RES_UP2) y += res[(((size_t)b * RH + hh / 2) * RW + ww / 2) * Cout + c];
          if (RES == BBDM_RES_DOWN2) {
            double a = 0;
            for (int dy = 0; dy < 2; ++dy)
              for (int dx = 0; dx < 2; ++dx) a += res[(((size_t)b * RH + 2 * hh + dy) * RW + 2 * ww + dx) * Cout + c];
            y += 0.25 * a;
          }
          const double got = out[(((size_t)b * H + hh) * W + ww) * Cout + c];
          worst = std::fmax(worst, std::fabs(got - y));
          scale = std::fmax(scale, std::fabs(y));
          w1[c] += got; w2[c] += got * got;
        }
  for (int c = 0; c < Cout; ++c) {
    r1 = std::fmax(r1, std::fabs(s1[c] - w1[c]) / (1.0 + std::fabs(w1[c])));
    r2 = std::fmax(r2, std::fabs(s2[c] - w2[c]) / (1.0 + std::fabs(w2[c])));
  }
  const bool ok = worst <= 2e-6 * scale && r1 < 1e-4 && r2 < 1e-4;
  std::printf("RES=%d B=%d H=%d W=%d Cout=%d bias=%d 1/s=%g: max abs dev %.3e (scale %.3e), partial sums %.1e / %.1e -> %s\n",
              RES, B, H, W, Cout, (int)with_bias, inv, worst, scale, r1, r2, ok ? "ok" : "FAIL");
  return ok ? 0 : 1;
}

int main() {
  int bad = 0;
  // 1/s of the weight planes: the all-zero default 2^-8 and the per-tensor scales of small / large weights
  // ragged maps (H or W not multiples of 6) exercise the masked edge tiles
  bad += run<BBDM_RES_NONE>(2, 12, 18, 64, true, 1.0f / 256);
  bad += run<BBDM_RES_NONE>(1, 7, 10, 128, false, 1.0f / 131072);
  bad += run<BBDM_RES_SAME>(2, 14, 12, 64, true, 1.0f / 8192);
  bad += run<BBDM_RES_SAME>(3, 16, 8, 128, false, 1.0f / 256);
  bad += run<BBDM_RES_UP2>(2, 8, 14, 64, true, 1.0f / 4096);
  bad += run<BBDM_RES_UP2>(1, 12, 12, 128, false, 1.0f / 256);
  bad += run<BBDM_RES_DOWN2>(2, 10, 12, 64, true, 1.0f / 256);
  bad += run<BBDM_RES_DOWN2>(1, 6, 8, 128, false, 1.0f / 16777216);
  std::printf(bad ? "FAILED\n" : "ALL OK\n");
  return bad;
}
