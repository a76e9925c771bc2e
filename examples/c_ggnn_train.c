/*
 * c_ggnn_train.c -- train one GGNN layer (GRU cell, 2 timesteps) from C: nothing but include/rgnn.h and the CUDA runtime.
 *
 * A seeded QM9-shaped batch: G = 8 molecules of 9 atoms (V = 72 nodes), L = 4 bond types with 40 bonds each, every bond
 * between two atoms of one molecule.  Node states h [V, D = 16] and a target [V, D].  Each step runs the two timesteps as
 * two rgnn_ggnn_forward calls (num_timesteps = 1, keeping each timestep's input), the squared loss
 * 0.5 * sum((y - target)^2) / V and its gradient (y - target) / V on the host, then rgnn_ggnn_backward from the last
 * timestep down, adding the two timesteps' weight gradients, and one SGD update of the edge weights W_l and the cell's
 * kernel, recurrent kernel and bias.  Prints the loss of each step, one per line.
 *
 *   gcc -std=c99 -O2 -I include -I /usr/local/cuda/include examples/c_ggnn_train.c \
 *       -L tf-gnn-samples_b200/lib -lrgnn -L /usr/local/cuda/lib64 -lcudart -o c_ggnn_train
 *   ./c_ggnn_train [steps]
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "rgnn.h"

enum { G = 8, ATOMS = 9, V = G * ATOMS, L = 4, E = 40, D = 16, T = 2 };
static const float LR = 0.1f;

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

/* w -= LR * (sum of the T timesteps' gradients) */
static void sgd(float* w, float* w_dev, float* const* g_dev, float* g_host, size_t n) {
  for (int t = 0; t < T; ++t) {
    download(g_host, g_dev[t], n);
    for (size_t i = 0; i < n; ++i) w[i] -= LR * g_host[i];
  }
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

  /* inputs, weights (host masters + device copies) and gradients (one set per timestep) */
  static float h[V * D], target[V * D], y[V * D], gy[V * D], w[L][D * D], kern[D * 3 * D], rec[D * 3 * D], bias[3 * D],
      scratch[D * 3 * D];
  fill_sym(h, V * D, 1.0f);
  for (int l = 0; l < L; ++l) fill_sym(w[l], D * D, 0.3f);
  fill_sym(kern, D * 3 * D, 0.3f);
  fill_sym(rec, D * 3 * D, 0.3f);
  fill_sym(bias, 3 * D, 0.1f);
  fill_sym(target, V * D, 1.0f);

  float* x_d[T + 1];   /* x_d[t]: input of timestep t; x_d[T]: the output */
  for (int t = 0; t <= T; ++t) x_d[t] = dev_alloc(V * D);
  float* g_d[2] = {dev_alloc(V * D), dev_alloc(V * D)};
  float *w_d[L], *gw_d[T][L], *gk_d[T], *gr_d[T], *gb_d[T];
  for (int l = 0; l < L; ++l) {
    w_d[l] = dev_alloc(D * D);
    upload(w_d[l], w[l], D * D);
  }
  for (int t = 0; t < T; ++t) {
    for (int l = 0; l < L; ++l) gw_d[t][l] = dev_alloc(D * D);
    gk_d[t] = dev_alloc(D * 3 * D);
    gr_d[t] = dev_alloc(D * 3 * D);
    gb_d[t] = dev_alloc(3 * D);
  }
  float* kern_d = dev_alloc(D * 3 * D);
  float* rec_d = dev_alloc(D * 3 * D);
  float* bias_d = dev_alloc(3 * D);
  upload(kern_d, kern, D * 3 * D);
  upload(rec_d, rec, D * 3 * D);
  upload(bias_d, bias, 3 * D);
  upload(x_d[0], h, V * D);

  const size_t fwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_GGNN, D, D, 0);
  const size_t bwd_bytes = rgnn_workspace_bytes(plan, RGNN_LAYER_GGNN_BACKWARD, D, D, 0);
  const size_t ws_bytes = fwd_bytes > bwd_bytes ? fwd_bytes : bwd_bytes;
  void* ws = NULL;
  CU(cudaMalloc(&ws, ws_bytes));
  const float* const* wc = (const float* const*)w_d;

  for (int step = 0; step < steps; ++step) {
    for (int t = 0; t < T; ++t)
      CK(rgnn_ggnn_forward(plan, x_d[t], D, D, wc, kern_d, rec_d, bias_d, RGNN_CELL_GRU, RGNN_ACT_TANH, RGNN_AGG_SUM, 1,
                           x_d[t + 1], ws, ws_bytes, stream));
    CU(cudaStreamSynchronize(stream));
    download(y, x_d[T], V * D);
    double loss = 0.0;
    for (int i = 0; i < V * D; ++i) {
      const double r = (double)y[i] - (double)target[i];
      loss += 0.5 * r * r / V;
      gy[i] = (float)(r / V);
    }
    printf("%.9g\n", loss);
    upload(g_d[0], gy, V * D);
    /* from the last timestep down: grad_out of timestep t is d_h of timestep t + 1 (d_h of timestep 0 is not needed) */
    for (int t = T - 1; t >= 0; --t)
      CK(rgnn_ggnn_backward(plan, x_d[t], D, wc, kern_d, rec_d, bias_d, RGNN_CELL_GRU, RGNN_ACT_TANH, RGNN_AGG_SUM,
                            g_d[(T - 1 - t) & 1], t > 0 ? g_d[(T - t) & 1] : NULL, gw_d[t], gk_d[t], gr_d[t], gb_d[t], ws,
                            ws_bytes, stream));
    CU(cudaStreamSynchronize(stream));
    for (int l = 0; l < L; ++l) {
      float* gl[T];
      for (int t = 0; t < T; ++t) gl[t] = gw_d[t][l];
      sgd(w[l], w_d[l], gl, scratch, D * D);
    }
    sgd(kern, kern_d, gk_d, scratch, D * 3 * D);
    sgd(rec, rec_d, gr_d, scratch, D * 3 * D);
    sgd(bias, bias_d, gb_d, scratch, 3 * D);
  }

  CK(rgnn_plan_destroy(plan));
  CU(cudaStreamSynchronize(stream));
  cudaFree(ws);
  for (int t = 0; t <= T; ++t) cudaFree(x_d[t]);
  cudaFree(g_d[0]); cudaFree(g_d[1]);
  cudaFree(kern_d); cudaFree(rec_d); cudaFree(bias_d);
  for (int l = 0; l < L; ++l) {
    cudaFree(w_d[l]);
    cudaFree(adj_dev[l]);
  }
  for (int t = 0; t < T; ++t) {
    for (int l = 0; l < L; ++l) cudaFree(gw_d[t][l]);
    cudaFree(gk_d[t]); cudaFree(gr_d[t]); cudaFree(gb_d[t]);
  }
  CU(cudaStreamDestroy(stream));
  return 0;
}
