// ia_union_find.cuh -- lock-free union-find over an int parent array, shared by the occupancy-grid build
// (ia_occupancy.cu) and the marching-cubes component pass (ia_mesh.cu).  Roots are the largest index of their set.
#pragma once

// find with path halving, for the union pass only.  There parent[x] >= x always holds (roots are the largest index),
// only roots are CAS-linked, and a halving write stores an ancestor into a non-root entry: a racy write can undo
// another thread's shortcut but never points a cell outside its tree.
static __device__ __forceinline__ int uf_find(int* parent, int i) {
    for (;;) {
        const int p = parent[i];
        if (p == i) return i;
        const int gp = parent[p];
        if (gp != p) parent[i] = gp;
        i = p;
    }
}

// roots are the largest linear index of the component (the label the reference's max-flood converges to)
static __device__ __forceinline__ void uf_union(int* parent, int a, int b) {
    for (;;) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicCAS(&parent[b], b, a);
        if (old == b) return;
        b = old;
    }
}

// read-only walk to the root, for the flatten pass.  Each thread of that pass stores its root into its own entry only,
// so every value a walk reads is an ancestor or the root.  A halving write here could replace a root that a finished
// thread had stored with a non-root ancestor, and a later pass would see that entry as belonging to another set.
static __device__ __forceinline__ int uf_root(const int* parent, int i) {
    for (;;) {
        const int p = parent[i];
        if (p == i) return i;
        i = p;
    }
}
