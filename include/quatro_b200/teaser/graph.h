// teaser/graph.h -- source-compatible replacement of the reference's include/teaser/graph.h:
//   class teaser::Graph            (reference include/teaser/graph.h:29-207)
//   class teaser::MaxCliqueSolver  (reference include/teaser/graph.h:219-274, src/graph.cc:12-130)
// Graph is a host-side adjacency list, as in the reference.  MaxCliqueSolver hands every graph to qb200_max_clique_batch_each
// (include/quatro_b200.h): the k-core peel and the clique search run on the device, a batch of graphs in one call.
// With the include path of INTEGRATION.md (Option A), #include "teaser/graph.h" resolves here.
#pragma once

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../quatro_b200.h"

namespace teaser {

// A simple undirected graph: vertices 0 .. numVertices() - 1, each with the list of its neighbours in insertion order.
class Graph {
 public:
  Graph() = default;

  // As in the reference: numVertices() = adj_list.size(), the keys are the vertices 0 .. size - 1 and their lists are taken as they
  // are, every edge expected under both of its vertices; numEdges() = half the total list length.  A key outside 0 .. size - 1 throws
  // std::out_of_range (the reference writes past its adjacency list there).  findMaxClique reads an edge listed under one vertex only
  // as an edge, and refuses a neighbour id outside the graph as it refuses a self-loop.
  explicit Graph(const std::map<int, std::vector<int>>& adj_list) {
    adj_list_.resize(adj_list.size());
    for (const auto& e : adj_list) {
      if (!hasVertex(e.first)) throw std::out_of_range("teaser::Graph: adjacency list key outside 0 .. size - 1");
      adj_list_[(size_t)e.first] = e.second;
      num_edges_ += e.second.size();
    }
    num_edges_ /= 2;
  }

  // A vertex with no edges; an id below numVertices() already exists and changes nothing.
  void addVertex(const int& id) {
    if (id >= numVertices()) adj_list_.resize((size_t)id + 1);
  }

  // numVertices() = num_vertices
  void populateVertices(const int& num_vertices) { adj_list_.resize((size_t)num_vertices); }

  bool hasEdge(const int& vertex_1, const int& vertex_2) const {
    if (!hasVertex(vertex_1) || !hasVertex(vertex_2)) return false;
    const std::vector<int>& nb = adj_list_[(size_t)vertex_1];
    return std::find(nb.begin(), nb.end(), vertex_2) != nb.end();
  }

  bool hasVertex(const int& vertex) const { return vertex >= 0 && vertex < numVertices(); }

  // An edge that exists already is not added again.  Both vertices must exist (std::out_of_range otherwise).
  void addEdge(const int& vertex_1, const int& vertex_2) {
    if (!hasVertex(vertex_1) || !hasVertex(vertex_2)) throw std::out_of_range("teaser::Graph::addEdge: vertex does not exist");
    if (hasEdge(vertex_1, vertex_2)) return;
    adj_list_[(size_t)vertex_1].push_back(vertex_2);
    adj_list_[(size_t)vertex_2].push_back(vertex_1);
    ++num_edges_;
  }

  // Removing an edge that does not exist changes nothing.
  void removeEdge(const int& vertex_1, const int& vertex_2) {
    if (!hasEdge(vertex_1, vertex_2)) return;
    std::vector<int>& a = adj_list_[(size_t)vertex_1];
    std::vector<int>& b = adj_list_[(size_t)vertex_2];
    a.erase(std::remove(a.begin(), a.end(), vertex_2), a.end());
    b.erase(std::remove(b.begin(), b.end(), vertex_1), b.end());
    --num_edges_;
  }

  int numVertices() const { return (int)adj_list_.size(); }
  int numEdges() const { return (int)num_edges_; }
  const std::vector<int>& getEdges(int id) const { return adj_list_[(size_t)id]; }
  std::vector<int> getVertices() const {
    std::vector<int> v((size_t)numVertices());
    for (int i = 0; i < numVertices(); ++i) v[(size_t)i] = i;
    return v;
  }
  std::vector<std::vector<int>> getAdjList() const { return adj_list_; }
  void reserve(const int& num_vertices) { adj_list_.reserve((size_t)num_vertices); }
  void clear() {
    adj_list_.clear();
    num_edges_ = 0;
  }

 private:
  std::vector<std::vector<int>> adj_list_;
  size_t num_edges_ = 0;
};

// Maximum cliques of Graphs on the device.  Membership is canonical: among several maximum cliques the same one is returned on every
// run (DESIGN.md 5.3), where pmc's choice depends on thread timing.  The solver's handle is created on first use for graphs of up to
// 4096 vertices and rebuilt once for up to QB200_MAX_CORR (32768); a larger graph throws std::invalid_argument.
class MaxCliqueSolver {
 public:
  enum class CLIQUE_SOLVER_MODE { PMC_EXACT = 0, PMC_HEU = 1, KCORE_HEU = 2 };

  struct Params {
    CLIQUE_SOLVER_MODE solver_mode = CLIQUE_SOLVER_MODE::PMC_EXACT;
    bool solve_exactly = true;              // deprecated: false = PMC_HEU whatever solver_mode says (src/graph.cc:15-17)
    double kcore_heuristic_threshold = 1;
    // seconds in the reference; a device search has no deterministic wall clock, so the batch call's default node limit
    // (QB200_DEFAULT_CLIQUE_NODE_LIMIT nodes per graph) bounds the PMC_EXACT search instead
    double time_limit = 3600;
  };

  MaxCliqueSolver() = default;
  MaxCliqueSolver(Params params) : params_(params) {}

  // the maximum clique of `graph`, in ascending vertex ids
  std::vector<int> findMaxClique(Graph graph) { return findMaxCliques(std::vector<Graph>{std::move(graph)})[0]; }

  // findMaxClique of every graph, in one batch call
  std::vector<std::vector<int>> findMaxCliques(const std::vector<Graph>& graphs) {
    const size_t n = graphs.size();
    std::vector<std::vector<int>> out(n);
    if (n == 0) return out;
    int max_L = 0;
    for (const Graph& g : graphs) max_L = std::max(max_L, g.numVertices());
    qb200_handle* h = handle_for(max_L);
    std::vector<std::vector<int32_t>> edges(n);
    std::vector<qb200_graph> desc(n);
    std::vector<qb200_params> params(n);
    for (size_t i = 0; i < n; ++i) {
      const Graph& g = graphs[i];
      // every listed neighbour: both orientations of an edge are one edge to the batch call, so an edge listed under one of its
      // vertices only (possible through the adjacency-list constructor) counts as well
      for (int u = 0; u < g.numVertices(); ++u)
        for (const int v : g.getEdges(u)) { edges[i].push_back(u); edges[i].push_back(v); }
      desc[i] = qb200_graph{edges[i].empty() ? nullptr : edges[i].data(), nullptr, (int64_t)(edges[i].size() / 2), g.numVertices(), 0};
      qb200_default_params(&params[i]);
      params[i].inlier_selection_mode = params_.solve_exactly ? (int32_t)params_.solver_mode : QB200_PMC_HEU;
      params[i].kcore_heuristic_threshold = params_.kcore_heuristic_threshold;
      params[i].max_clique_node_limit = 0;
    }
    const int cap = std::max(max_L, 1);
    std::vector<int32_t> cliques(n * (size_t)cap);
    std::vector<qb200_result> res(n);
    qb200_pair_lists lists;
    std::memset(&lists, 0, sizeof(lists));
    lists.cap_per_pair = cap;
    lists.kind = QB200_MEM_HOST;
    lists.clique = cliques.data();
    const int rc = qb200_max_clique_batch_each(h, desc.data(), (int32_t)n, params.data(), QB200_MEM_HOST, res.data(), &lists);
    if (rc < 0) throw std::runtime_error(std::string("qb200_max_clique_batch_each: ") + qb200_last_error(h));
    for (size_t i = 0; i < n; ++i) {
      if (res[i].status < 0)
        throw std::invalid_argument("teaser::MaxCliqueSolver: graph " + std::to_string(i) +
                                    " has a self-loop or an edge to a vertex beyond numVertices()");
      const int32_t* c = cliques.data() + i * (size_t)cap;
      out[i].assign(c, c + res[i].clique_size);
    }
    return out;
  }

 private:
  struct HandleDeleter {
    void operator()(qb200_handle* h) const { qb200_destroy(h); }
  };

  // the solver's handle, able to hold graphs of L vertices: 8 graphs of up to 4096 vertices per wave, or one of up to QB200_MAX_CORR;
  // the front-end capacities are the smallest qb200_create takes (a graph batch reads no scans)
  qb200_handle* handle_for(int L) {
    if (L > QB200_MAX_CORR)
      throw std::invalid_argument("teaser::MaxCliqueSolver: a graph of " + std::to_string(L) + " vertices exceeds the device capacity (" +
                                  std::to_string(QB200_MAX_CORR) + ")");
    if (handle_ && L <= handle_corr_) return handle_.get();
    const int corr = L <= 4096 ? 4096 : QB200_MAX_CORR;
    handle_.reset();  // release the old workspaces before allocating the larger ones
    qb200_config cfg;
    qb200_default_config(&cfg);
    cfg.max_batch_slots = corr == 4096 ? 8 : 1;
    cfg.max_raw_points = 1;
    cfg.max_voxel_points = 128;
    cfg.max_corr = corr;
    qb200_handle* h = nullptr;
    const int st = qb200_create(&cfg, &h);
    if (st != QB200_OK)
      throw std::runtime_error("qb200_create failed (status " + std::to_string(st) + "): no usable CUDA device; there is no CPU fallback");
    handle_ = std::shared_ptr<qb200_handle>(h, HandleDeleter());
    handle_corr_ = corr;
    return h;
  }

  Params params_;
  std::shared_ptr<qb200_handle> handle_;  // shared by copies of the solver, like the reference's plain members
  int handle_corr_ = 0;
};

}  // namespace teaser
