#pragma once
#include "common.cuh"
namespace b200 {
// powerset classes of N <= 32 speakers with at most M per frame, in utils/powerset.py's order: set size 0 .. M,
// itertools.combinations within each size.  mask[c] holds the speakers of class c (bit j = speaker j).
constexpr int kPowersetMaxClasses = 32;
struct PowersetMap {
  int K = 0, N = 0;
  unsigned mask[kPowersetMaxClasses] = {};
};
// builds the map; returns false (and sets the error message) when N / M is out of range or the class count exceeds 32
bool powerset_map(int N, int M, PowersetMap* map);
int powerset_to_multilabel(const unsigned char* cls, long long n, const PowersetMap& map, unsigned char* ml,
                           cudaStream_t stream);
int speaker_count(const unsigned char* seg, const int* sf, int C, int F, unsigned char* count, cudaStream_t stream);
int reconstruct(const unsigned char* seg, const signed char* hard, const int* sf, int C, int F, int Kout,
                const unsigned char* count, unsigned char* out, cudaStream_t stream);
int frame_transitions(const unsigned char* discrete, int F, int K, int cap, int* buf, cudaStream_t stream);
int aggregate_scores(const float* scores, const int* sf, int C, int F, int nf, int K, const double* hamming,
                     const double* warm, int skip_average, float missing, float epsilon, float* out,
                     cudaStream_t stream);
int powerset_speech(const unsigned char* cls, long long n, const PowersetMap& map, float* out, cudaStream_t stream);
int push_bytes(const void* src, long long bytes, void* const* dsts, int n, cudaStream_t stream);
int clean_frames(const unsigned char* seg, int C, int* clean, unsigned char* active, cudaStream_t stream);
}
