// heap.cuh -- std::priority_queue's push and pop as libstdc++ implements them, over an array of node ids ordered by a
// per-node key that may change while an id sits in the heap.  Shared by the A* search (astar.cu, NodeComparator0 over
// f_score) and the local tour's Dijkstra search (local_tour.cu, NodeCompare over g_value_): both compare
// node1 > node2 through the key each id holds at the moment of the comparison.
#pragma once

namespace {

// std::priority_queue<NodePtr, vector, NodeComparator0>::push / pop as libstdc++ implements them (push_heap,
// pop_heap -> __adjust_heap -> __push_heap), comparing node1->f_score > node2->f_score through the current f of each id
__device__ void heap_sift_up(int* heap, const double* f, int hole, int v) {
  const double fv = f[v];
  int parent = (hole - 1) / 2;
  while (hole > 0 && f[heap[parent]] > fv) {
    heap[hole] = heap[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  heap[hole] = v;
}
__device__ void heap_pop(int* heap, int len, const double* f) {
  if (len <= 1) return;
  const int n = len - 1;
  const int v = heap[n];
  heap[n] = heap[0];
  int hole = 0, child = 0;
  while (child < (n - 1) / 2) {
    child = 2 * (child + 1);
    if (f[heap[child]] > f[heap[child - 1]]) child--;
    heap[hole] = heap[child];
    hole = child;
  }
  if ((n & 1) == 0 && child == (n - 2) / 2) {
    child = 2 * (child + 1);
    heap[hole] = heap[child - 1];
    hole = child - 1;
  }
  heap_sift_up(heap, f, hole, v);
}

}  // namespace
