#pragma once
#include "common.cuh"
namespace b200 {
// problems of at least this many observations take the whole-GPU linkage path (packed distances allocated per call);
// smaller ones the batched one-CTA-per-problem kernel with a dense matrix in the workspace
constexpr int kLinkGridMinDefault = 32769;
constexpr int kLinkMaxRows = 1048560;          // 65535 tiles of 16 rows in the distance kernel's grid
size_t linkage_workspace_bytes_batched(const int* row_offsets, int nfiles, int dim, int grid_min);
size_t linkage_grid_bytes(const int* row_offsets, int nfiles, int grid_min);
int linkage_centroid_batched(const double* x, const int* row_offsets, int nfiles, int dim, int normalize, double* Z,
                             void* ws, cudaStream_t st, int grid_min);
int plda_transform(const double* x, int n, int Din, int Dout, int L, const double* mean1, const double* mean2,
                   const double* lda, const double* mu, const double* trT, double* fea, cudaStream_t st);
int weighted_centroids(const double* q, int n, int S, const int* kept, int K, const double* train, int dim,
                       double* centroids, cudaStream_t st);
int cdist_cosine(const double* a, int m, const double* b, int k, int dim, double* d, cudaStream_t st);
size_t vbx_workspace_bytes_batched(const int* n, const int* S, int nfiles, int D);
int vbx_run_batched(const double* fea, const double* phi, const int* n, const int* S, int nfiles, int D, double Fa,
                    double Fb, int max_iters, double epsilon, double* gamma, double* pi, int* iters_host, void* ws,
                    cudaStream_t st);
int assign_clusters(const double* soft, int C, int K, int constrained, signed char* hard, cudaStream_t st);
int fcluster_distance(const double* Z, int n, double t, int* T);
}
