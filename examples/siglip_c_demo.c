/*
 * Plain-C use of the C ABI (include/siglip_b200.h): no Python, no torch.
 * One rank, B x D random unit-norm embeddings (bf16), fused forward + backward, checked against a double-precision
 * host evaluation of the same formula (reference: distributed_sigmoid_loss.py:22-33,47).
 *
 *   nvcc -o siglip_c_demo examples/siglip_c_demo.c -Iinclude -Ldistributed_sigmoid_loss_b200 -lsiglip_b200 \
 *        -Xlinker -rpath -Xlinker $PWD/distributed_sigmoid_loss_b200
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "siglip_b200.h"

static uint16_t f32_to_bf16(float f) { /* round to nearest even */
  uint32_t u;
  memcpy(&u, &f, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static float bf16_to_f32(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static double softplus(double x) { return x > 0 ? x + log1p(exp(-x)) : log1p(exp(x)); }

#define CHECK_CUDA(x)                                                            \
  do {                                                                           \
    cudaError_t e_ = (x);                                                        \
    if (e_ != cudaSuccess) {                                                     \
      fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_));                   \
      return 2;                                                                  \
    }                                                                            \
  } while (0)
#define CHECK_SIGLIP(x)                                                          \
  do {                                                                           \
    if ((x) != 0) {                                                              \
      fprintf(stderr, "%s: %s\n", #x, siglip_last_error());                      \
      return 3;                                                                  \
    }                                                                            \
  } while (0)

int main(void) {
  const int B = 384, D = 128;
  const float t_prime = logf(10.0f), bias = -10.0f;
  printf("%s, %d sm_90 device(s)\n", siglip_version(), siglip_device_count());
  if (siglip_device_count() == 0) {
    fprintf(stderr, "no H100: this library has no CPU fallback\n");
    return 1;
  }
  const size_t n = (size_t)B * D;
  uint16_t* h_img = (uint16_t*)malloc(n * 2);
  uint16_t* h_txt = (uint16_t*)malloc(n * 2);
  srand(7);
  for (int which = 0; which < 2; ++which) {
    uint16_t* dst = which ? h_txt : h_img;
    for (int i = 0; i < B; ++i) {
      double row[1024], ss = 0;
      for (int d = 0; d < D; ++d) {
        row[d] = (double)rand() / RAND_MAX - 0.5;
        ss += row[d] * row[d];
      }
      for (int d = 0; d < D; ++d) dst[(size_t)i * D + d] = f32_to_bf16((float)(row[d] / sqrt(ss)));
    }
  }
  void *d_img, *d_txt;
  float *d_scal, *d_dimg, *d_dtxt; /* d_scal: t', bias, loss, dt', dbias */
  CHECK_CUDA(cudaMalloc(&d_img, n * 2));
  CHECK_CUDA(cudaMalloc(&d_txt, n * 2));
  CHECK_CUDA(cudaMalloc((void**)&d_scal, 5 * sizeof(float)));
  CHECK_CUDA(cudaMalloc((void**)&d_dimg, n * sizeof(float)));
  CHECK_CUDA(cudaMalloc((void**)&d_dtxt, n * sizeof(float)));
  const float h_scal[2] = {t_prime, bias};
  CHECK_CUDA(cudaMemcpy(d_img, h_img, n * 2, cudaMemcpyHostToDevice));
  CHECK_CUDA(cudaMemcpy(d_txt, h_txt, n * 2, cudaMemcpyHostToDevice));
  CHECK_CUDA(cudaMemcpy(d_scal, h_scal, sizeof(h_scal), cudaMemcpyHostToDevice));

  siglip_ctx* ctx = NULL;
  CHECK_SIGLIP(siglip_ctx_create(&ctx, 0, 0, 1, B, D));
  CHECK_SIGLIP(siglip_fwd_bwd(ctx, d_img, d_txt, d_scal + 0, d_scal + 1, d_scal + 2, d_dimg, d_dtxt, d_scal + 3,
                              d_scal + 4, NULL));
  CHECK_CUDA(cudaDeviceSynchronize());
  float out[5];
  float* h_dimg = (float*)malloc(n * sizeof(float));
  CHECK_CUDA(cudaMemcpy(out, d_scal, sizeof(out), cudaMemcpyDeviceToHost));
  CHECK_CUDA(cudaMemcpy(h_dimg, d_dimg, n * sizeof(float), cudaMemcpyDeviceToHost));

  /* host evaluation in double */
  const double t = exp((double)t_prime);
  double loss = 0, dbias = 0, dtp = 0, err2 = 0, ref2 = 0;
  double* dimg = (double*)calloc(n, sizeof(double));
  for (int i = 0; i < B; ++i)
    for (int j = 0; j < B; ++j) {
      double s = 0;
      for (int d = 0; d < D; ++d) s += (double)bf16_to_f32(h_img[(size_t)i * D + d]) * bf16_to_f32(h_txt[(size_t)j * D + d]);
      const double z = t * s + bias, y = (i == j) ? 1.0 : -1.0;
      loss += softplus(-y * z);
      const double g = -y / (1.0 + exp(y * z)); /* d softplus(-y z) / dz */
      dbias += g;
      dtp += g * s;
      for (int d = 0; d < D; ++d) dimg[(size_t)i * D + d] += g * bf16_to_f32(h_txt[(size_t)j * D + d]);
    }
  loss /= B;
  dbias /= B;
  dtp *= t / B;
  for (size_t k = 0; k < n; ++k) {
    const double r = dimg[k] * t / B, e = h_dimg[k] - r;
    err2 += e * e;
    ref2 += r * r;
  }
  const double e_loss = fabs(out[2] - loss) / fabs(loss), e_dtp = fabs(out[3] - dtp) / fabs(dtp),
               e_db = fabs(out[4] - dbias) / fabs(dbias), e_dimg = sqrt(err2 / ref2);
  printf("loss %.6f (host %.6f)  rel errors: loss %.1e dt' %.1e dbias %.1e dimg %.1e\n", out[2], loss, e_loss, e_dtp,
         e_db, e_dimg);
  siglip_ctx_destroy(ctx);
  const int ok = e_loss < 1e-3 && e_dtp < 1e-3 && e_db < 1e-3 && e_dimg < 1e-3;
  printf(ok ? "C-ABI DEMO PASS\n" : "C-ABI DEMO FAIL\n");
  return ok ? 0 : 4;
}
