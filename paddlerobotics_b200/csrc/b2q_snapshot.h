// b2q_snapshot.h — what the env and learner snapshots (b2q_snapshot_*, b2q_sac_snapshot_*) share: the fixed-size header slot at the
// start of a blob, the kernel that stores a host-built header into it (a kernel argument is copied at launch, so a save needs neither a
// host sync nor a staging buffer), the field-by-field header comparison of a load and a byte hash.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace b2q_snap {

constexpr size_t HDR_BYTES = 1024;     // header slot at the start of every blob; the payload follows it, 16-byte aligned
struct HdrWords { uint32_t w[HDR_BYTES / 4]; };

static __global__ void write_header_kernel(HdrWords h, uint32_t* dst) {
  for (int i = threadIdx.x; i < (int)(HDR_BYTES / 4); i += blockDim.x) dst[i] = h.w[i];
}
// stores hdr (a trivially copyable struct of at most HDR_BYTES) into the first HDR_BYTES of dst, zero-padded
template <typename H>
inline cudaError_t write_header(const H& hdr, void* dst, cudaStream_t s) {
  static_assert(sizeof(H) <= HDR_BYTES, "snapshot header outgrew its slot");
  HdrWords w;
  std::memset(&w, 0, sizeof w);
  std::memcpy(&w, &hdr, sizeof(H));
  write_header_kernel<<<1, 128, 0, s>>>(w, static_cast<uint32_t*>(dst));
  return cudaGetLastError();
}

// one header field: its name (for the error message), offset and size; compared bytewise, so doubles must match bit for bit
struct Field { const char* name; size_t off, size; };
// the first field in which a and b differ, or nullptr
inline const char* first_difference(const void* a, const void* b, const Field* f, int n) {
  for (int i = 0; i < n; i++)
    if (std::memcmp(static_cast<const char*>(a) + f[i].off, static_cast<const char*>(b) + f[i].off, f[i].size) != 0) return f[i].name;
  return nullptr;
}

inline uint64_t fnv1a(const void* p, size_t n, uint64_t h = 1469598103934665603ull) {
  const unsigned char* c = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < n; i++) { h ^= c[i]; h *= 1099511628211ull; }
  return h;
}

}  // namespace b2q_snap
