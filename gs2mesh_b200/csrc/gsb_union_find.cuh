// Lock-free union-find, the undirected edge key and its sort width, shared by the mesh cluster kernels (gsb_mesh.cu)
// and the topology queries (gsb_topology.cu); the union-find also joins DBSCAN's core points (gsb_normals.cu).
//
// Union-find over int ids in the style of ECL-CC: a larger root is always hooked under a smaller one with atomicCAS, so
// parent[x] <= x holds at every moment and the surviving root of a set is its smallest id.  Parents are read with
// relaxed atomic loads; finds halve the path they walk.  Only roots are ever CAS'd and a non-root never becomes a root
// again, so a path-halving store (an ancestor into a non-root) cannot undo a hook.
#pragma once

#include <cuda/atomic>

namespace gsb {

using ParentRef = cuda::atomic_ref<int, cuda::thread_scope_device>;

__device__ __forceinline__ int uf_load(int* parent, int x) { return ParentRef(parent[x]).load(cuda::memory_order_relaxed); }

__device__ __forceinline__ int uf_find(int* parent, int x) {
  int p = uf_load(parent, x);
  while (p != x) {
    const int gp = uf_load(parent, p);
    if (gp != p) ParentRef(parent[x]).store(gp, cuda::memory_order_relaxed);
    x = gp;
    p = uf_load(parent, x);
  }
  return x;
}

__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  a = uf_find(parent, a);
  b = uf_find(parent, b);
  while (a != b) {
    if (a < b) {
      const int s = a;
      a = b;
      b = s;
    }
    const int old = atomicCAS(&parent[a], a, b);  // hook the larger root under the smaller
    if (old == a) return;
    a = uf_find(parent, old);  // a was hooked elsewhere in the meantime
    b = uf_find(parent, b);
  }
}

// The root of x once every union has finished (a later kernel): a plain walk, no stores.
__device__ __forceinline__ int uf_root(const int* parent, int x) {
  int p = parent[x];
  while (p != x) {
    x = p;
    p = parent[x];
  }
  return x;
}

// The key of the undirected edge (a, b): min * stride + max with stride = n_vertices + 1, Open3D's GetOrderedEdge as one
// integer.  Degenerate edges (a, a) get keys like any other; keys < stride^2.
__device__ __forceinline__ unsigned long long edge_key(long long a, long long b, unsigned long long stride) {
  const unsigned long long lo = (unsigned long long)(a < b ? a : b), hi = (unsigned long long)(a < b ? b : a);
  return lo * stride + hi;
}

// The number of low bits a radix sort of keys <= max_value needs.
inline int bits_of(unsigned long long max_value) {
  int b = 0;
  while (b < 64 && (max_value >> b) != 0) ++b;
  return b;
}

}  // namespace gsb
