// A caller of SurfelMapping::setPointLabels / getPointLabels (include/suma_b200.hpp). Reads raw scans (uint32 n, then
// n*4 floats), processes them with the records on and writes the records of the last scan to argv[3] as raw bytes.
#include <cstdio>
#include <vector>

#include "suma_b200.hpp"

using namespace suma;

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  int width = std::atoi(argv[2]);
  ParameterList params;
  params.insert("data_width", width);
  params.insert("model_width", width);
  params.insert("max iterations", 10);
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
  SurfelMapping fusion(params);
  std::vector<sb_point_label> rec;
  fusion.setPointLabels(true);
  try {
    fusion.getPointLabels(rec);  // no scan yet: refused
    return 5;
  } catch (const std::runtime_error&) {
  }
  for (const Laserscan& s : scans) fusion.processScan(s);
  fusion.getPointLabels(rec);
  FILE* o = std::fopen(argv[3], "wb");
  if (!o || std::fwrite(rec.data(), sizeof(sb_point_label), rec.size(), o) != rec.size()) return 6;
  std::fclose(o);
  std::printf("records %zu size %zu\n", rec.size(), sizeof(sb_point_label));
  return 0;
}
