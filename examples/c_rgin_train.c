/*
 * c_rgin_train.c -- train one RGIN layer from C: nothing but include/rgnn.h and the CUDA runtime.
 *
 * A seeded QM9-shaped batch: G = 8 molecules of 9 atoms (V = 72 nodes), L = 4 bond types with 40 bonds each, every bond
 * between two atoms of one molecule.  Node states h [V, D = 16] and a target [V, D].  The layer is the reference's default
 * RGIN: source-only messages through a per-type edge MLP with one hidden layer, ReLU, sum aggregation, no aggregation MLP,
 * then the layer norm.  Each step runs rgnn_rgin_forward (num_timesteps = 1), the squared loss
 * 0.5 * sum((y - target)^2) / V and its gradient (y - target) / V on the host, then rgnn_rgin_backward and one SGD update of
 * the edge-MLP kernels and the layer-norm gamma / beta.  Prints the loss of each step, one per line.
 *
 *   gcc -std=c99 -O2 -I include -I /usr/local/cuda/include examples/c_rgin_train.c \
 *       -L tf-gnn-samples_b200/lib -lrgnn -L /usr/local/cuda/lib64 -lcudart -o c_rgin_train
 *   ./c_rgin_train [steps]
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "rgnn.h"

enum { G = 8, ATOMS = 9, V = G * ATOMS, L = 4, E = 40, D = 16, HIDDEN = 1, NE = HIDDEN + 1 };
static const float LR = 0.2f;

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

  /* the graph: bonds (source, target) of each type, both atoms in one molecule */
  static int32_t adj_host[L][E][2];
  int32_t* adj_dev[L];
  int64_t num_edges[L];
  for (int l = 0; l < L; ++l) {
    for (int e = 0; e < E; ++e) {
      const int g = (int)(uniform() * G);
      adj_host[l][e][0] = (int32_t)(g * ATOMS + (int)(uniform() * ATOMS));
      adj_host[l][e][1] = (int32_t)(g * ATOMS + (int)(uniform() * ATOMS));
    }
    void* p = NULL;
    CU(cudaMalloc(&p, sizeof(adj_host[l])));
    CU(cudaMemcpy(p, adj_host[l], sizeof(adj_host[l]), cudaMemcpyHostToDevice));
    adj_dev[l] = (int32_t*)p;
    num_edges[l] = E;
  }
  rgnn_plan_t* plan = NULL;
  CK(rgnn_plan_create(&plan, V, L, (const int32_t* const*)adj_dev, num_edges, stream));

  /* inputs and weights (host masters + device copies); edge-MLP kernels type-major: entry l * NE + j is layer j of type l */
  static float h[V * D], target[V * D], y[V * D], gy[V * D], ew[L * NE][D * D], gamma[D], beta[D], scratch[D * D];
  fill_sym(h, V * D, 1.0f);
  for (int i = 0; i < L * NE; ++i) fill_sym(ew[i], D * D, 0.5f);
  for (int i = 0; i < D; ++i) gamma[i] = 1.0f + 0.2f * (2.0f * uniform() - 1.0f);
  fill_sym(beta, D, 0.2f);
  fill_sym(target, V * D, 1.0f);
  const int32_t dims[NE + 1] = {D, D, D};

  float* x_d = dev_alloc(V * D);
  float* y_d = dev_alloc(V * D);
  float* g_d = dev_alloc(V * D);
  float *ew_d[L * NE], *gew_d[L * NE];
  for (int i = 0; i < L * NE; ++i) {
    ew_d[i] = dev_alloc(D * D);
    gew_d[i] = dev_alloc(D * D);
    upload(ew_d[i], ew[i], D * D);
  }
  float* gamma_d = dev_alloc(D);
  float* beta_d = dev_alloc(D);
  float* ggamma_d = dev_alloc(D);
  float* gbeta_d = dev_alloc(D);
  upload(gamma_d, gamma, D);
  upload(beta_d, beta, D);
  upload(x_d, h, V * D);

  const size_t fwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_RGIN, D, D, NE);
  const size_t bwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_RGIN_BACKWARD, D, D, NE);
  const size_t ws_bytes = fwd_bytes > bwd_bytes ? fwd_bytes : bwd_bytes;
  void* ws = NULL;
  CU(cudaMalloc(&ws, ws_bytes));
  const float* const* ewc = (const float* const*)ew_d;

  for (int step = 0; step < steps; ++step) {
    CK(rgnn_rgin_forward(plan, x_d, D, D, ewc, dims, HIDDEN, NULL, NULL, -1, gamma_d, beta_d, RGNN_ACT_RELU, RGNN_AGG_SUM, 0, 1,
                         y_d, ws, ws_bytes, stream));
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
    CK(rgnn_rgin_backward(plan, x_d, D, D, ewc, dims, HIDDEN, NULL, NULL, -1, gamma_d, beta_d, RGNN_ACT_RELU, RGNN_AGG_SUM, 0,
                          g_d, NULL, gew_d, NULL, ggamma_d, gbeta_d, ws, ws_bytes, stream));
    CU(cudaStreamSynchronize(stream));
    for (int i = 0; i < L * NE; ++i) sgd(ew[i], ew_d[i], gew_d[i], scratch, D * D);
    sgd(gamma, gamma_d, ggamma_d, scratch, D);
    sgd(beta, beta_d, gbeta_d, scratch, D);
  }

  CK(rgnn_plan_destroy(plan));
  CU(cudaStreamSynchronize(stream));
  cudaFree(ws);
  cudaFree(x_d); cudaFree(y_d); cudaFree(g_d);
  cudaFree(gamma_d); cudaFree(beta_d); cudaFree(ggamma_d); cudaFree(gbeta_d);
  for (int i = 0; i < L * NE; ++i) {
    cudaFree(ew_d[i]);
    cudaFree(gew_d[i]);
  }
  for (int l = 0; l < L; ++l) cudaFree(adj_dev[l]);
  CU(cudaStreamDestroy(stream));
  return 0;
}
