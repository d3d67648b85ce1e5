// Host build of the feature store's row-index table (fs_row_table, similari_b200/csrc/sb_fstore.cuh): the code fstore.cu
// runs on the host for every search / associate call, compiled as it is for tests/test_feature_store_io_cpu.py.
#include "../../similari_b200/csrc/sb_fstore.cuh"

// row_src has room for offs[Q] entries, qoff for Q + 1; returns the rows that take part
extern "C" int shim_fs_row_table(int Q, const int32_t* offs, int K, int* row_src, int* qoff) {
  std::vector<int> src, off;
  sb::fs_row_table(Q, offs, K, &src, &off);
  std::copy(src.begin(), src.end(), row_src);
  std::copy(off.begin(), off.end(), qoff);
  return (int)src.size();
}
