// Error statistics of the MUFU approximations used by the FAC recursion against double precision
// (nvcc -gencode arch=compute_90a,code=sm_90a scripts/mufu_bias.cu -o build/mufu_bias):
//   part 1: lg2.approx(1 + r) on r in [0,1], ex2.approx(d) on d in [-30,0], and the composite lg2(1 + ex2(d))
//   part 2: the composite the recursion actually evaluates, F(d) = lg2.approx(fma(ex2.approx(d), 1.25, 1.25)) against
//           log2(1.25 (1 + 2^d)), binned by its argument q' = 1.25 (1 + 2^d) in [1.25, 2.5]
#include <cstdio>
#include <cmath>
#include <cuda_runtime.h>
__global__ void k(int n, float* lgv, float* exv, float* lsev, float* cmp, float* cmpq) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float r = (float)i / (float)(n - 1);
  float q = 1.0f + r, y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(q));
  lgv[i] = y;
  float d = -30.0f * (float)i / (float)(n - 1), e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(d));
  exv[i] = e;
  float q2 = 1.0f + e, y2;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y2) : "f"(q2));
  lsev[i] = y2;
  // part 2: d spread so that q' covers [1.25, 2.5] evenly: d = log2(q'/1.25 - 1)
  float qt = 1.25f + 1.25f * (float)i / (float)(n - 1);
  float dd = log2f(fmaxf(qt / 1.25f - 1.0f, 1e-30f)), e2, y3;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e2) : "f"(dd));
  float q3 = fmaf(e2, 1.25f, 1.25f);
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y3) : "f"(q3));
  cmp[i] = y3;
  cmpq[i] = dd;
}
int main() {
  const int n = 1 << 20;
  float *a, *b, *c, *f, *g;
  cudaMallocManaged(&a, n * 4); cudaMallocManaged(&b, n * 4); cudaMallocManaged(&c, n * 4); cudaMallocManaged(&f, n * 4); cudaMallocManaged(&g, n * 4);
  k<<<(n + 255) / 256, 256>>>(n, a, b, c, f, g);
  cudaDeviceSynchronize();
  const int nb = 16;
  double sl[nb] = {0}, se[nb] = {0}, sc[nb] = {0}, al[nb] = {0}, ac[nb] = {0};
  for (int i = 0; i < n; ++i) {
    float r = (float)i / (float)(n - 1);
    float q = 1.0f + r;
    double el = (double)a[i] - log2((double)q);
    float d = -30.0f * (float)i / (float)(n - 1);
    double ee = ((double)b[i] - exp2((double)d)) / exp2((double)d);
    double ec = (double)c[i] - log2(1.0 + exp2((double)d));
    int bin = i * nb / n;
    sl[bin] += el; al[bin] += fabs(el); se[bin] += ee; sc[bin] += ec; ac[bin] += fabs(ec);
  }
  printf("bin  r-range lg2(1+r): mean err, mean |err| ;  d-range ex2: mean rel err ; lse(d)=lg2(1+ex2(d)): mean err, mean |err|\n");
  for (int j = 0; j < nb; ++j)
    printf("%2d  r~%.3f  %+.3e %.3e   d~%6.2f  %+.3e   %+.3e %.3e\n", j, (j + 0.5) / nb, sl[j] / (n / nb), al[j] / (n / nb), -30.0 * (j + 0.5) / nb,
           se[j] / (n / nb), sc[j] / (n / nb), ac[j] / (n / nb));
  const int nb2 = 40;
  double s2[nb2] = {0}, ss2[nb2] = {0};
  int cnt[nb2] = {0};
  for (int i = 0; i < n; ++i) {
    double dd = (double)g[i];
    double qe = 1.25 * (1.0 + exp2(dd));
    double err = (double)f[i] - log2(qe);
    int bin = (int)((qe - 1.25) / 1.25 * nb2);
    if (bin < 0) bin = 0;
    if (bin >= nb2) bin = nb2 - 1;
    s2[bin] += err; ss2[bin] += err * err; cnt[bin]++;
  }
  printf("composite F(d) = lg2.approx(fma(ex2.approx(d), 1.25, 1.25)) - log2(1.25 (1 + 2^d)), binned by q' (mean, std)\n");
  for (int j = 0; j < nb2; ++j) {
    double m = s2[j] / cnt[j];
    printf("q'~%.4f  %+.3e  %.3e\n", 1.25 + 1.25 * (j + 0.5) / nb2, m, sqrt(fmax(0.0, ss2[j] / cnt[j] - m * m)));
  }
  return 0;
}
