/*
 * c_rgat_train.c -- train one RGAT layer from C: nothing but include/rgnn.h and the CUDA runtime.
 *
 * A seeded random graph (V = 64 nodes, L = 2 edge types, 256 edges each), node states h [V, D = 16] and a target
 * [V, D], H = 2 attention heads.  Each step: y = rgnn_rgat_forward(h), the squared loss 0.5 * sum((y - target)^2) / V and
 * its gradient (y - target) / V on the host, rgnn_rgat_backward for the gradients of every weight, and one SGD update of
 * the edge weights W_l and the attention vectors a_l.  Prints the loss of each step, one per line.
 *
 *   gcc -std=c99 -O2 -I include -I /usr/local/cuda/include examples/c_rgat_train.c \
 *       -L tf-gnn-samples_b200/lib -lrgnn -L /usr/local/cuda/lib64 -lcudart -o c_rgat_train
 *   ./c_rgat_train [steps]
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "rgnn.h"

enum { V = 64, L = 2, E = 256, D = 16, H = 2 };
static const float LR = 0.05f;

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
static void sgd(float* w, float* w_dev, float* g_dev, float* g_host, size_t n) {
  download(g_host, g_dev, n);
  for (size_t i = 0; i < n; ++i) w[i] -= LR * g_host[i];
  upload(w_dev, w, n);
}

int main(int argc, char** argv) {
  const int steps = argc > 1 ? atoi(argv[1]) : 8;
  cudaStream_t stream;
  CU(cudaStreamCreate(&stream));

  /* the graph: edge (source, target) pairs of each type */
  static int32_t adj_host[L][E][2];
  int32_t* adj_dev[L];
  int64_t num_edges[L];
  for (int l = 0; l < L; ++l) {
    for (int e = 0; e < E; ++e) {
      adj_host[l][e][0] = (int32_t)(uniform() * V);
      adj_host[l][e][1] = (int32_t)(uniform() * V);
    }
    void* p = NULL;
    CU(cudaMalloc(&p, sizeof(adj_host[l])));
    CU(cudaMemcpy(p, adj_host[l], sizeof(adj_host[l]), cudaMemcpyHostToDevice));
    adj_dev[l] = (int32_t*)p;
    num_edges[l] = E;
  }
  rgnn_plan_t* plan = NULL;
  CK(rgnn_plan_create(&plan, V, L, (const int32_t* const*)adj_dev, num_edges, stream));

  /* inputs, weights (host masters + device copies) and gradients */
  static float h[V * D], target[V * D], y[V * D], gy[V * D], w[L][D * D], att[L][2 * D], scratch[D * D];
  fill_sym(h, V * D, 1.0f);
  for (int l = 0; l < L; ++l) fill_sym(w[l], D * D, 0.5f);
  for (int l = 0; l < L; ++l) fill_sym(att[l], 2 * D, 0.5f);
  fill_sym(target, V * D, 1.0f);

  float* h_d = dev_alloc(V * D);
  float* y_d = dev_alloc(V * D);
  float* gy_d = dev_alloc(V * D);
  float *w_d[L], *att_d[L], *gw_d[L], *gatt_d[L];
  for (int l = 0; l < L; ++l) {
    w_d[l] = dev_alloc(D * D);
    att_d[l] = dev_alloc(2 * D);
    gw_d[l] = dev_alloc(D * D);
    gatt_d[l] = dev_alloc(2 * D);
    upload(w_d[l], w[l], D * D);
    upload(att_d[l], att[l], 2 * D);
  }
  upload(h_d, h, V * D);

  const size_t fwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_RGAT, D, D, 0);
  const size_t bwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_RGAT_BACKWARD, D, D, 0);
  const size_t ws_bytes = fwd_bytes > bwd_bytes ? fwd_bytes : bwd_bytes;
  void* ws = NULL;
  CU(cudaMalloc(&ws, ws_bytes));

  for (int step = 0; step < steps; ++step) {
    CK(rgnn_rgat_forward(plan, h_d, D, D, (const float* const*)w_d, (const float* const*)att_d, H, RGNN_ACT_TANH, 1, y_d,
                         ws, ws_bytes, stream));
    CU(cudaStreamSynchronize(stream));
    download(y, y_d, V * D);
    double loss = 0.0;
    for (int i = 0; i < V * D; ++i) {
      const double r = (double)y[i] - (double)target[i];
      loss += 0.5 * r * r / V;
      gy[i] = (float)(r / V);
    }
    printf("%.9g\n", loss);
    upload(gy_d, gy, V * D);
    CK(rgnn_rgat_backward(plan, h_d, D, D, (const float* const*)w_d, (const float* const*)att_d, H, RGNN_ACT_TANH, gy_d,
                          NULL, gw_d, gatt_d, ws, ws_bytes, stream));
    CU(cudaStreamSynchronize(stream));
    for (int l = 0; l < L; ++l) {
      sgd(w[l], w_d[l], gw_d[l], scratch, D * D);
      sgd(att[l], att_d[l], gatt_d[l], scratch, 2 * D);
    }
  }

  CK(rgnn_plan_destroy(plan));
  CU(cudaStreamSynchronize(stream));
  cudaFree(ws);
  cudaFree(h_d); cudaFree(y_d); cudaFree(gy_d);
  for (int l = 0; l < L; ++l) {
    cudaFree(w_d[l]); cudaFree(att_d[l]); cudaFree(gw_d[l]); cudaFree(gatt_d[l]);
    cudaFree(adj_dev[l]);
  }
  CU(cudaStreamDestroy(stream));
  return 0;
}
