// vampnet_b200 — the one cache of constant device tables (the spectrogram's FFT tables and mel banks, the beat
// tracker's tables, the pitch shift's DFT bases).  A table is built on the host once per (device, key), uploaded into
// one allocation and kept for the life of the process, so a call after the first costs a lookup under one mutex.
#include <map>
#include <mutex>
#include <utility>

#include "kernels.h"

namespace vnb {

cudaError_t device_table(const std::vector<double>& key, const std::function<std::vector<char>()>& build,
                         const char** dev) {
  static std::mutex mu;
  static std::map<std::pair<int, std::vector<double>>, const char*> tables;
  int d = 0;
  cudaError_t e = cudaGetDevice(&d);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  auto it = tables.find({d, key});
  if (it == tables.end()) {
    const std::vector<char> host = build();
    char* p = nullptr;
    if ((e = cudaMalloc(&p, host.size())) != cudaSuccess) return e;
    if ((e = cudaMemcpy(p, host.data(), host.size(), cudaMemcpyHostToDevice)) != cudaSuccess) {
      cudaFree(p);
      return e;
    }
    it = tables.emplace(std::make_pair(d, key), p).first;
  }
  *dev = it->second;
  return cudaSuccess;
}

}  // namespace vnb
