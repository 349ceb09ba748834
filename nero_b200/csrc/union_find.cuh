// Connected components by union-find on the GPU: uf_init makes every element its own root, the caller's hook kernel calls
// uf_unite once per edge, and uf_flatten's rounds of pointer jumping leave parent[v] = the root of v = the smallest index of
// its component, so the labels do not depend on scheduling.
#pragma once
#include <cuda_runtime.h>

namespace nero {

// root of x with path halving.  Every parent pointer points to a smaller (or the same) index and only ever moves to an
// ancestor, so the halving stores, racing with each other and with the hooks, keep a forest with the same roots.
__device__ __forceinline__ int uf_find(volatile int* parent, int x) {
  while (true) {
    const int p = parent[x];
    if (p == x) return x;
    const int g = parent[p];
    if (g != p) parent[x] = g;
    x = g;
  }
}

__device__ __forceinline__ void uf_unite(int* parent, int a, int b) {
  volatile int* vp = parent;
  while (true) {
    a = uf_find(vp, a);
    b = uf_find(vp, b);
    if (a == b) return;
    if (a > b) { const int s = a; a = b; b = s; }
    // hook root b under the smaller root a; if b stopped being a root meanwhile, retry from its new parent
    const int old = atomicCAS(parent + b, b, a);
    if (old == b) return;
    b = old;
  }
}

// The library's files are compiled separately without relocatable device code, so each one gets its own copy of the kernels.
namespace {

constexpr int kUfThreads = 256;

__global__ void __launch_bounds__(kUfThreads) uf_init_kernel(int* __restrict__ parent, long long m) {
  const long long v = (long long)blockIdx.x * kUfThreads + threadIdx.x;
  if (v < m) parent[v] = int(v);
}

// one round of pointer jumping: parent[v] <- parent[parent[v]].  Reading a value another thread has already jumped only
// moves further up, so after k rounds parent[v] is at least the 2^k-th ancestor of v, or the root.
__global__ void __launch_bounds__(kUfThreads) uf_jump_kernel(int* parent, long long m) {
  const long long v = (long long)blockIdx.x * kUfThreads + threadIdx.x;
  if (v >= m) return;
  volatile int* vp = parent;
  const int p = vp[v];
  const int g = vp[p];
  if (g != p) vp[v] = g;
}

// parent[v] = v for the m elements: one launch
void uf_init(int* parent, long long m, cudaStream_t stream) {
  uf_init_kernel<<<unsigned((m + kUfThreads - 1) / kUfThreads), kUfThreads, 0, stream>>>(parent, m);
}

// ceil(log2 m) + 1 rounds of pointer jumping, which flatten any tree of depth < m (every tree of m elements) onto its root.
// Launches unchecked: the caller checks its launches together.
void uf_flatten(int* parent, long long m, cudaStream_t stream) {
  int rounds = 1;
  while ((1LL << (rounds - 1)) < m) ++rounds;
  for (int r = 0; r < rounds; ++r) uf_jump_kernel<<<unsigned((m + kUfThreads - 1) / kUfThreads), kUfThreads, 0, stream>>>(parent, m);
}

}  // namespace

}  // namespace nero
