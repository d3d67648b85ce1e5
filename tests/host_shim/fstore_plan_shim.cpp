// Host build of the feature store blob's section plan (fs_blob_sections, similari_b200/csrc/sb_fstore.cuh): the code
// save and load run on the host for every blob, compiled as it is for tests/test_feature_store_io_cpu.py.
#include <cstdio>

#include "../../similari_b200/csrc/sb_fstore.cuh"

// Writes up to `cap` sections (name into names[i * 32], bytes, role, class index); returns how many the plan has.
extern "C" int shim_fs_blob_sections(int version, uint64_t live, int K, int stype, int gate, int keep, int n,
                                     const int32_t* dims, uint64_t hist_total, int cap, char* names, uint64_t* bytes,
                                     int* role, int* cls) {
  const std::vector<sb::FsSection> plan = sb::fs_blob_sections(version, live, K, stype, gate, keep, n, dims, hist_total);
  for (int i = 0; i < (int)plan.size() && i < cap; ++i) {
    snprintf(names + 32 * i, 32, "%s", plan[i].name);
    bytes[i] = plan[i].bytes;
    role[i] = plan[i].role;
    cls[i] = plan[i].cls;
  }
  return (int)plan.size();
}
