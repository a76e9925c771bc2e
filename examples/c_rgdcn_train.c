/*
 * c_rgdcn_train.c -- train one RGDCN layer from C: nothing but include/rgnn.h and the CUDA runtime.
 *
 * A seeded QM9-shaped batch: G = 8 molecules of 9 atoms (V = 72 nodes), L = 4 bond types with 40 bonds each, every bond
 * between two atoms of one molecule.  Node states h [V, D = 128] and a target [V, D].  The layer has the reference model's
 * defaults: C = 8 channels of K = 16, per-channel kernel inputs, untied channel kernels, ReLU, sum aggregation, messages
 * normalised by the per-type in-degree.  Each step runs rgnn_rgdcn_forward (num_timesteps = 1), the squared loss
 * 0.5 * sum((y - target)^2) / V and its gradient (y - target) / V on the host, then rgnn_rgdcn_backward and one SGD update of
 * the L * C channel kernels [K, K * K].  Prints the loss of each step, one per line.
 *
 *   gcc -std=c99 -O2 -I include -I /usr/local/cuda/include examples/c_rgdcn_train.c \
 *       -L tf-gnn-samples_b200/lib -lrgnn -L /usr/local/cuda/lib64 -lcudart -o c_rgdcn_train
 *   ./c_rgdcn_train [steps]
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "rgnn.h"

enum { G = 8, ATOMS = 9, V = G * ATOMS, L = 4, E = 40, C = 8, K = 16, D = C * K, NK = L * C };
static const float LR = 0.5f;

#define CK(call)                                                                         \
  do {                                                                                   \
    int rc_ = (call);                                                                    \
    if (rc_ != RGNN_OK) {                                                                \
      fprintf(stderr, "%s failed (%d): %s\n", #call, rc_, rgnn_last_error());            \
      exit(1);                                                                           \
    }                                                                                    \
  } while (0)
#define CU(call)                                                                         \
  do {                                                                                   \
    cudaError_t e_ = (call);                                                             \
    if (e_ != cudaSuccess) {                                                             \
      fprintf(stderr, "%s failed: %s\n", #call, cudaGetErrorString(e_));                 \
      exit(1);                                                                           \
    }                                                                                    \
  } while (0)

/* x <- 1664525 x + 1013904223 (mod 2^32); uniform in [0, 1) from the top 24 bits */
static uint32_t rng_state = 12345u;
static float uniform(void) {
  rng_state = 1664525u * rng_state + 1013904223u;
  return (float)(rng_state >> 8) * (1.0f / 16777216.0f);
}
static void fill_sym(float* x, int n, float scale) {
  for (int i = 0; i < n; ++i) x[i] = (2.0f * uniform() - 1.0f) * scale;
}

static float* dev_alloc(size_t n) {
  void* p = NULL;
  CU(cudaMalloc(&p, n * sizeof(float)));
  return (float*)p;
}
static void upload(float* dst, const float* src, size_t n) { CU(cudaMemcpy(dst, src, n * sizeof(float), cudaMemcpyHostToDevice)); }
static void download(float* dst, const float* src, size_t n) { CU(cudaMemcpy(dst, src, n * sizeof(float), cudaMemcpyDeviceToHost)); }

/* w -= LR * gradient */
static void sgd(float* w, float* w_dev, const float* g_dev, float* g_host, size_t n) {
  download(g_host, g_dev, n);
  for (size_t i = 0; i < n; ++i) w[i] -= LR * g_host[i];
  upload(w_dev, w, n);
}

int main(int argc, char** argv) {
  const int steps = argc > 1 ? atoi(argv[1]) : 8;
  cudaStream_t stream;
  CU(cudaStreamCreate(&stream));

  /* the graph: bonds (source, target) of each type, both atoms in one molecule; in-degrees per type [L, V] */
  static int32_t adj_host[L][E][2];
  static float num_incoming[L * V];
  int32_t* adj_dev[L];
  int64_t num_edges[L];
  for (int l = 0; l < L; ++l) {
    for (int e = 0; e < E; ++e) {
      const int g = (int)(uniform() * G);
      adj_host[l][e][0] = (int32_t)(g * ATOMS + (int)(uniform() * ATOMS));
      adj_host[l][e][1] = (int32_t)(g * ATOMS + (int)(uniform() * ATOMS));
      num_incoming[l * V + adj_host[l][e][1]] += 1.0f;
    }
    void* p = NULL;
    CU(cudaMalloc(&p, sizeof(adj_host[l])));
    CU(cudaMemcpy(p, adj_host[l], sizeof(adj_host[l]), cudaMemcpyHostToDevice));
    adj_dev[l] = (int32_t*)p;
    num_edges[l] = E;
  }
  rgnn_plan_t* plan = NULL;
  CK(rgnn_plan_create(&plan, V, L, (const int32_t* const*)adj_dev, num_edges, stream));

  /* inputs and kernels (host masters + device copies); channel kernels type-major: entry l * C + c is channel c of type l */
  static float h[V * D], target[V * D], y[V * D], gy[V * D], fw[NK][K * K * K], scratch[K * K * K];
  fill_sym(h, V * D, 1.0f);
  for (int i = 0; i < NK; ++i) fill_sym(fw[i], K * K * K, 0.4f);
  fill_sym(target, V * D, 1.0f);

  float* x_d = dev_alloc(V * D);
  float* y_d = dev_alloc(V * D);
  float* g_d = dev_alloc(V * D);
  float* cnt_d = dev_alloc(L * V);
  float *fw_d[NK], *gfw_d[NK];
  for (int i = 0; i < NK; ++i) {
    fw_d[i] = dev_alloc(K * K * K);
    gfw_d[i] = dev_alloc(K * K * K);
    upload(fw_d[i], fw[i], K * K * K);
  }
  upload(x_d, h, V * D);
  upload(cnt_d, num_incoming, L * V);

  const size_t fwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_RGDCN, D, D, K);
  const size_t bwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_RGDCN_BACKWARD, D, D, K);
  const size_t ws_bytes = fwd_bytes > bwd_bytes ? fwd_bytes : bwd_bytes;
  void* ws = NULL;
  CU(cudaMalloc(&ws, ws_bytes));
  const float* const* fwc = (const float* const*)fw_d;

  for (int step = 0; step < steps; ++step) {
    CK(rgnn_rgdcn_forward(plan, x_d, D, C, fwc, 0, cnt_d, RGNN_ACT_RELU, RGNN_AGG_SUM, 1, 1, y_d, ws, ws_bytes, stream));
    CU(cudaStreamSynchronize(stream));
    download(y, y_d, V * D);
    double loss = 0.0;
    for (int i = 0; i < V * D; ++i) {
      const double r = (double)y[i] - (double)target[i];
      loss += 0.5 * r * r / V;
      gy[i] = (float)(r / V);
    }
    printf("%.9g\n", loss);
    upload(g_d, gy, V * D);
    /* d_h is not needed: the input states are not trained */
    CK(rgnn_rgdcn_backward(plan, x_d, D, C, fwc, 0, 0, cnt_d, RGNN_ACT_RELU, RGNN_AGG_SUM, 1, g_d, NULL, gfw_d, ws, ws_bytes,
                           stream));
    CU(cudaStreamSynchronize(stream));
    for (int i = 0; i < NK; ++i) sgd(fw[i], fw_d[i], gfw_d[i], scratch, K * K * K);
  }

  CK(rgnn_plan_destroy(plan));
  CU(cudaStreamSynchronize(stream));
  cudaFree(ws);
  cudaFree(x_d); cudaFree(y_d); cudaFree(g_d); cudaFree(cnt_d);
  for (int i = 0; i < NK; ++i) {
    cudaFree(fw_d[i]);
    cudaFree(gfw_d[i]);
  }
  for (int l = 0; l < L; ++l) cudaFree(adj_dev[l]);
  CU(cudaStreamDestroy(stream));
  return 0;
}
