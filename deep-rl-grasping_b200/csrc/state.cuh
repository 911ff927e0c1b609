// Training-state files (state.cu): the container format every learner's b2g_*_state_save / _load shares, and the steps of a
// load they have in common.
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

#include <functional>
#include <string>
#include <vector>

namespace b2g {

enum : uint32_t { STATE_KIND_SAC = 1, STATE_KIND_BDQ = 2, STATE_KIND_DQN = 3, STATE_KIND_PPO = 4, STATE_KIND_TRPO = 5 };

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
inline StatePiece host_piece(void* p, size_t bytes) { StatePiece s; s.host = p; s.bytes = bytes; return s; }
inline StatePiece dev_piece(void* p, size_t bytes) { StatePiece s; s.dev = p; s.bytes = bytes; return s; }

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

// ---- the sections every learner's file starts with: HOST (its host bookkeeping) and CNTR (its device counters), then PARM
// (n_param floats of the parameter arena), ADMM and ADMV (n_moments floats of the Adam moments)
std::vector<StateSection> host_sections(void* host, size_t host_bytes, void* counters, size_t counter_bytes);
std::vector<StateSection> adam_sections(float* P, size_t n_param, float* Mo, float* Vo, size_t n_moments);

// ---- the load steps every learner shares.  A learner's file holds the host sections HOST and CNTR, then its device sections.
// The file's tags are HOST, CNTR and those of dev, in order (B2G_EINVAL naming the learner otherwise).
int state_check_tags(const StateReader& rd, const std::vector<StateSection>& dev, const char* learner);
// Section 2 + i of the file is as long as dev[i], for every i.
int state_check_lengths(const StateReader& rd, const std::vector<StateSection>& dev);
// Streams sections 2.. into dev, then runs restore(), which puts back what the handle keeps outside them.  *broken is set before
// the first write and cleared once restore() has succeeded: a handle that failed part way accepts only destroy and load.
int state_read_device(StateReader& rd, const std::vector<StateSection>& dev, bool* broken, const std::function<int()>& restore);

// ---- VecNormalize's obs_rms: a handle that owns it writes one more fingerprint field (obs_rms = 1) and one more section (ORMS:
// count, then mean[E] and var[E] as float64); one that does not reads and writes the files it always did.
std::vector<FpField> fp_with_rms(std::vector<FpField> fp, bool owns_rms);
StateSection rms_section(double* count, double* mean, double* var, int E);
// rd.open() with the fingerprint of a handle that owns obs_rms or not; a file that differs in that alone is refused with a
// message naming rms_set_call, the call that gives a handle its obs_rms.
int state_open_rms(StateReader& rd, const char* path, uint32_t kind, const std::vector<FpField>& fp, bool owns_rms, const char* rms_set_call);
// 1 when the fingerprint of the state file at path has a field of that name, 0 when not, -1 when it is no readable state file
// of that handle kind
int state_fp_field(const char* path, uint32_t kind, const char* name);

}  // namespace b2g
