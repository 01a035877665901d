// Checkpoint and resume through the C++ mirror's file overloads: reads raw scans (uint32 n, then n*4 floats), processes
// the first N, saves the session to a file, loads it into a new SurfelMapping and processes the rest. Prints the final
// pose and the surfel count.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "suma_b200.hpp"

using namespace suma;

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  const int width = std::atoi(argv[2]);
  const size_t n_first = static_cast<size_t>(std::atoi(argv[3]));
  const std::string state = argv[4];
  ParameterList params;
  params.insert("data_width", width);
  params.insert("model_width", width);
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  std::vector<Laserscan> scans;
  for (;;) {
    uint32_t n = 0;
    if (std::fread(&n, 4, 1, f) != 1) break;
    Laserscan s;
    s.points.resize(static_cast<size_t>(n) * 4);
    if (std::fread(s.points.data(), 4, s.points.size(), f) != s.points.size()) return 4;
    scans.push_back(s);
  }
  std::fclose(f);
  {
    SurfelMapping first(params);
    for (size_t i = 0; i < n_first && i < scans.size(); ++i) first.processScan(scans[i]);
    first.saveState(state);
  }
  SurfelMapping resumed(params);
  resumed.loadState(state);
  for (size_t i = n_first; i < scans.size(); ++i) resumed.processScan(scans[i]);
  Matrix4d pose = resumed.getCurrentPose();
  std::printf("pose");
  for (int i = 0; i < 16; ++i) std::printf(" %.17g", pose.m[i]);
  std::printf("\nsurfels %u timestamp %u\n", resumed.getMap()->size(), resumed.timestamp());
  bool refused = false;
  try {
    resumed.loadState(std::vector<uint8_t>(16, 0));
  } catch (const std::runtime_error&) {
    refused = true;
  }
  std::printf("refused %d\n", refused ? 1 : 0);
  return 0;
}
