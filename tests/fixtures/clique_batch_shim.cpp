// GPU check of the teaser/graph.h shim: Graphs built with addEdge, solved one by one with findMaxClique and all at once with
// findMaxCliques, and again through the adjacency-list constructor; all must agree.
//   clique_batch_shim graphs.txt     first line "n_graphs mode kcore_threshold", then per graph "L m" and m lines "u v"
// Prints "clique <size> <ids...>" per graph and "edges <numEdges()>" before it; exit 1 if the single and batch results differ, 4 if the
// adjacency-list copy differs.
#include <fstream>
#include <iostream>

#include "teaser/graph.h"

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  std::ifstream in(argv[1]);
  int n = 0, mode = 0;
  double thr = 1.0;
  in >> n >> mode >> thr;
  std::vector<teaser::Graph> graphs((size_t)n);
  for (teaser::Graph& g : graphs) {
    int L = 0;
    long long m = 0;
    in >> L >> m;
    g.populateVertices(L);
    for (long long k = 0; k < m; ++k) {
      int u = 0, v = 0;
      in >> u >> v;
      g.addEdge(u, v);
    }
  }
  try {
    teaser::MaxCliqueSolver::Params params;
    params.solver_mode = static_cast<teaser::MaxCliqueSolver::CLIQUE_SOLVER_MODE>(mode);
    params.kcore_heuristic_threshold = thr;
    teaser::MaxCliqueSolver solver(params);
    const std::vector<std::vector<int>> batch = solver.findMaxCliques(graphs);
    int rc = 0;
    for (size_t i = 0; i < graphs.size(); ++i) {
      const std::vector<int> one = solver.findMaxClique(graphs[i]);
      if (one != batch[i]) rc = 1;
      std::map<int, std::vector<int>> lists;  // the same graph through the adjacency-list constructor
      for (int u = 0; u < graphs[i].numVertices(); ++u) lists[u] = graphs[i].getEdges(u);
      const teaser::Graph copy(lists);
      if (copy.numVertices() != graphs[i].numVertices() || copy.numEdges() != graphs[i].numEdges() || solver.findMaxClique(copy) != one)
        rc = 4;
      std::cout << "edges " << graphs[i].numEdges() << "\nclique " << one.size();
      for (const int v : one) std::cout << " " << v;
      std::cout << "\n";
    }
    return rc;
  } catch (const std::exception& e) {
    std::cerr << "exception: " << e.what() << std::endl;
    return 3;
  }
}
