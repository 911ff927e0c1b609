// Training-state files (state.cu): the container format b2g_sac_state_save / _load and b2g_bdq_state_save / _load share.
//
// Layout (little-endian):
//   StateHeader                  magic "B2GSTATE", format version, handle kind, field / section counts, total file size
//   FpField[n_fp]                configuration fingerprint: named integer or real fields; a load compares them one by one
//   SecEntry[n_sec]              per section: tag, offset, length, checksum of its bytes
//   section data                 contiguous, in table order
// Device-resident sections are streamed through two pinned chunk buffers on a copy stream, so the copy of chunk k + 1 overlaps
// the file I/O of chunk k and neither host memory nor the device ever holds a second full copy of the replay.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

namespace b2g {

enum : uint32_t { STATE_KIND_SAC = 1, STATE_KIND_BDQ = 2, STATE_KIND_DQN = 3, STATE_KIND_PPO = 4 };

constexpr uint32_t state_tag(const char (&s)[5]) {
  return (uint32_t)(unsigned char)s[0] | (uint32_t)(unsigned char)s[1] << 8 | (uint32_t)(unsigned char)s[2] << 16 |
         (uint32_t)(unsigned char)s[3] << 24;
}

struct FpField {
  char name[31];
  char kind;        // 'i': v is an int64, 'f': v holds the bits of a double
  uint64_t v;
};
FpField fp_int(const char* name, int64_t v);
FpField fp_real(const char* name, double v);

// A contiguous piece of a section: host memory (host != nullptr) or device memory.
struct StatePiece {
  void* host = nullptr;
  void* dev = nullptr;
  size_t bytes = 0;
};
struct StateSection {
  uint32_t tag = 0;
  std::vector<StatePiece> pieces;
  size_t bytes() const;
};

// Writes the whole file.  Device pieces must be quiescent (the caller has synchronised the streams that write them).
int state_write(const char* path, uint32_t kind, const std::vector<FpField>& fp, const std::vector<StateSection>& secs);

// Reading: open() checks the header, the fingerprint (B2G_EINVAL naming the first field that differs), the section table and
// the file size without touching any handle state.  read_host() reads a whole section into host memory and verifies its
// checksum; read_pieces() streams one into host / device pieces and verifies the checksum once the bytes have landed.
class StateReader {
 public:
  ~StateReader();
  int open(const char* path, uint32_t kind, const std::vector<FpField>& fp);
  int n_sections() const { return (int)tags_.size(); }
  uint32_t tag(int i) const { return tags_[i]; }
  uint64_t bytes(int i) const { return lens_[i]; }
  int read_host(int i, void* dst, size_t bytes);
  int read_pieces(int i, const std::vector<StatePiece>& pieces);

 private:
  FILE* f_ = nullptr;
  std::string path_;
  std::vector<uint32_t> tags_;
  std::vector<uint64_t> offs_, lens_, sums_;
};

}  // namespace b2g
