// The reference README's "How do I just use the Core API?" program (README.md:74-100), against libefusion.so.
// Usage: core_api_example <raw.klg> <width> <height> <fx> <fy> <cx> <cy> [lookahead]  -> prints the final pose and surfel
// count. With `lookahead` the log is read one frame ahead and the next frame is handed to processFrame as well.
#include <ElasticFusion.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 8) return 2;
  const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
  Resolution::getInstance(w, h);
  Intrinsics::getInstance((float)std::atof(argv[4]), (float)std::atof(argv[5]), (float)std::atof(argv[6]), (float)std::atof(argv[7]));
  // open loop, as `ElasticFusion -o` configures it (MainController.cpp:179-183)
  ElasticFusion eFusion(2147483647 / 2, 35000, 5e-05, 1e-05, false, false, false, 115, 10, 3, 10, false, 0.3095, true, false, "/tmp/ef_b200_example",
                        500000);
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  int32_t numFrames = 0;
  if (std::fread(&numFrames, 4, 1, f) != 1) return 4;
  const bool lookahead = argc > 8;
  std::vector<uint8_t> rgb[2] = {std::vector<uint8_t>((size_t)w * h * 3), std::vector<uint8_t>((size_t)w * h * 3)};
  std::vector<uint16_t> depth[2] = {std::vector<uint16_t>((size_t)w * h), std::vector<uint16_t>((size_t)w * h)};
  int64_t ts[2];
  auto readFrame = [&](int slot) -> int {
    int32_t dsz, isz;
    if (std::fread(&ts[slot], 8, 1, f) != 1 || std::fread(&dsz, 4, 1, f) != 1 || std::fread(&isz, 4, 1, f) != 1) return 5;
    if (dsz != w * h * 2 || isz != w * h * 3) return 6;  // raw payloads only (Tools/RawLogReader.cpp:80-97)
    if (std::fread(depth[slot].data(), 1, dsz, f) != (size_t)dsz || std::fread(rgb[slot].data(), 1, isz, f) != (size_t)isz) return 7;
    return 0;
  };
  if (numFrames > 0)
    if (int rc = readFrame(0)) return rc;
  for (int i = 0; i < numFrames; ++i) {
    const int cur = i & 1, nxt = cur ^ 1;
    const bool haveNext = i + 1 < numFrames;
    if (haveNext)
      if (int rc = readFrame(nxt)) return rc;
    if (lookahead && haveNext)
      eFusion.processFrame(rgb[cur].data(), depth[cur].data(), ts[cur], 1.0f, nullptr, rgb[nxt].data(), depth[nxt].data());
    else
      eFusion.processFrame(rgb[cur].data(), depth[cur].data(), ts[cur], 1.0f);
  }
  std::fclose(f);
  const auto T = eFusion.get_T_wc().matrix();
  std::printf("POSE");
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) std::printf(" %.9f", (double)T(r, c));
  std::printf("\nCOUNT %u TICK %d\n", eFusion.getGlobalModel().lastCount(), eFusion.getTick());
  // ElasticFusion::savePly (Core/ElasticFusion.cpp:684-781) with a threshold the few frames of a test log can pass
  eFusion.setConfidenceThreshold(0.9f);
  eFusion.savePly();
  return 0;
}
