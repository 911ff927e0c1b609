// Training-state files: container format, checksums and the streamed device <-> file copies (layout in state.cuh).
#include <cuda_runtime.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>

#include "host.cuh"
#include "state.cuh"

namespace b2g {
namespace {

constexpr char kMagic[8] = {'B', '2', 'G', 'S', 'T', 'A', 'T', 'E'};
constexpr uint32_t kVersion = 1;
constexpr size_t kChunk = 64ull << 20;     // bytes per pinned staging buffer (two of them)

struct StateHeader {
  char magic[8];
  uint32_t version, kind, n_fp, n_sec;
  uint64_t file_bytes;
};
struct SecEntry {
  uint32_t tag, pad;
  uint64_t offset, bytes, checksum;
};
static_assert(sizeof(StateHeader) == 32 && sizeof(FpField) == 40 && sizeof(SecEntry) == 32, "file layout");

// 64-bit checksum over a byte stream fed in pieces of any size: four independent multiply-rotate lanes over 32-byte blocks
// (fast enough to keep up with the copies), the lanes folded together with the length and the trailing bytes at the end.
class Hasher {
 public:
  void update(const void* p, size_t n) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    total_ += n;
    if (npend_) {
      const size_t k = std::min(n, (size_t)32 - npend_);
      memcpy(pend_ + npend_, b, k);
      npend_ += k; b += k; n -= k;
      if (npend_ < 32) return;
      block(pend_);
      npend_ = 0;
    }
    for (; n >= 32; b += 32, n -= 32) block(b);
    memcpy(pend_, b, n);
    npend_ = n;
  }
  uint64_t digest() const {
    uint64_t h = rotl(l_[0], 1) + rotl(l_[1], 7) + rotl(l_[2], 12) + rotl(l_[3], 18);
    for (uint64_t x : l_) h = (h ^ round(0, x)) * P1 + P4;
    h += total_;
    for (size_t i = 0; i < npend_; ++i) h = rotl(h ^ (pend_[i] * P5), 11) * P1;
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
  }

 private:
  static constexpr uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull,
                            P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
  static uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
  static uint64_t round(uint64_t acc, uint64_t w) { return rotl(acc + w * P2, 31) * P1; }
  void block(const unsigned char* b) {
    uint64_t w[4];
    memcpy(w, b, 32);
    for (int i = 0; i < 4; ++i) l_[i] = round(l_[i], w[i]);
  }
  uint64_t l_[4] = {P1 + P2, P2, 0, 0ull - P1};
  unsigned char pend_[32]{};
  size_t npend_ = 0;
  uint64_t total_ = 0;
};

// Two pinned chunk buffers and a copy stream; every pending copy is waited for before destruction.
struct Staging {
  unsigned char* buf[2]{};
  cudaEvent_t ev[2]{};
  cudaStream_t s = nullptr;
  size_t chunk = 0;
  ~Staging() {
    if (s) cudaStreamSynchronize(s);
    for (int k = 0; k < 2; ++k) {
      if (buf[k]) cudaFreeHost(buf[k]);
      if (ev[k]) cudaEventDestroy(ev[k]);
    }
    if (s) cudaStreamDestroy(s);
  }
  int init(size_t largest) {
    chunk = std::min(kChunk, (largest + 4095) / 4096 * 4096);
    if (chunk == 0) return 0;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (int k = 0; k < 2; ++k) {
      CK(cudaHostAlloc((void**)&buf[k], chunk, cudaHostAllocDefault));
      CK(cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming));
    }
    return 0;
  }
};

size_t largest_dev_piece(const std::vector<StateSection>& secs) {
  size_t m = 0;
  for (const auto& s : secs)
    for (const auto& p : s.pieces) if (!p.host) m = std::max(m, p.bytes);
  return m;
}

int io_fail(const std::string& what, const std::string& path) {
  return b2g_fail(B2G_EINVAL, what + " (" + path + "): " + strerror(errno));
}

std::string fp_value(const FpField& f) {
  if (f.kind == 'f') {
    double d;
    memcpy(&d, &f.v, sizeof d);
    char b[64];
    snprintf(b, sizeof b, "%.9g", d);
    return b;
  }
  return std::to_string((int64_t)f.v);
}

}  // namespace

FpField fp_int(const char* name, int64_t v) {
  FpField f{};
  snprintf(f.name, sizeof f.name, "%s", name);
  f.kind = 'i';
  f.v = (uint64_t)v;
  return f;
}
FpField fp_real(const char* name, double v) {
  FpField f{};
  snprintf(f.name, sizeof f.name, "%s", name);
  f.kind = 'f';
  memcpy(&f.v, &v, sizeof v);
  return f;
}

size_t StateSection::bytes() const {
  size_t n = 0;
  for (const auto& p : pieces) n += p.bytes;
  return n;
}

int state_write(const char* path, uint32_t kind, const std::vector<FpField>& fp, const std::vector<StateSection>& secs) {
  if (!path) return b2g_fail(B2G_EINVAL, "state file path is NULL");
  StateHeader hd{};
  memcpy(hd.magic, kMagic, 8);
  hd.version = kVersion; hd.kind = kind; hd.n_fp = (uint32_t)fp.size(); hd.n_sec = (uint32_t)secs.size();
  std::vector<SecEntry> tab(secs.size());
  uint64_t off = sizeof(StateHeader) + fp.size() * sizeof(FpField) + secs.size() * sizeof(SecEntry);
  for (size_t i = 0; i < secs.size(); ++i) {
    tab[i].tag = secs[i].tag; tab[i].offset = off; tab[i].bytes = secs[i].bytes();
    off += tab[i].bytes;
  }
  hd.file_bytes = off;
  Staging st;
  if (int rc = st.init(largest_dev_piece(secs))) return rc;
  FILE* f = fopen(path, "wb");
  if (!f) return io_fail("cannot create the state file", path);
  struct Closer { FILE*& f; ~Closer() { if (f) fclose(f); } } closer{f};
  const long table_at = (long)(sizeof(StateHeader) + fp.size() * sizeof(FpField));
  if (fwrite(&hd, sizeof hd, 1, f) != 1 || (!fp.empty() && fwrite(fp.data(), sizeof(FpField), fp.size(), f) != fp.size()) ||
      (!tab.empty() && fwrite(tab.data(), sizeof(SecEntry), tab.size(), f) != tab.size()))
    return io_fail("cannot write the state header", path);
  for (size_t i = 0; i < secs.size(); ++i) {
    Hasher hs;
    for (const StatePiece& p : secs[i].pieces) {
      if (p.host) {
        hs.update(p.host, p.bytes);
        if (p.bytes && fwrite(p.host, 1, p.bytes, f) != p.bytes) return io_fail("cannot write the state file", path);
        continue;
      }
      // device piece: the copy of chunk k + 1 is in flight while chunk k is hashed and written
      const size_t n_chunks = (p.bytes + st.chunk - 1) / st.chunk;
      auto issue = [&](size_t k) -> int {
        const size_t o = k * st.chunk, n = std::min(st.chunk, p.bytes - o);
        CK(cudaMemcpyAsync(st.buf[k & 1], (const unsigned char*)p.dev + o, n, cudaMemcpyDeviceToHost, st.s));
        CK(cudaEventRecord(st.ev[k & 1], st.s));
        return 0;
      };
      if (n_chunks) if (int rc = issue(0)) return rc;
      for (size_t k = 0; k < n_chunks; ++k) {
        if (k + 1 < n_chunks) if (int rc = issue(k + 1)) return rc;
        CK(cudaEventSynchronize(st.ev[k & 1]));
        const size_t n = std::min(st.chunk, p.bytes - k * st.chunk);
        hs.update(st.buf[k & 1], n);
        if (fwrite(st.buf[k & 1], 1, n, f) != n) return io_fail("cannot write the state file", path);
      }
    }
    tab[i].checksum = hs.digest();
  }
  if (fseek(f, table_at, SEEK_SET) != 0 || (!tab.empty() && fwrite(tab.data(), sizeof(SecEntry), tab.size(), f) != tab.size()) ||
      fflush(f) != 0 || fsync(fileno(f)) != 0)
    return io_fail("cannot finish the state file", path);
  const int rc = fclose(f);
  f = nullptr;
  if (rc != 0) return io_fail("cannot close the state file", path);
  return 0;
}

StateReader::~StateReader() {
  if (f_) fclose(f_);
}

int StateReader::open(const char* path, uint32_t kind, const std::vector<FpField>& fp) {
  if (!path) return b2g_fail(B2G_EINVAL, "state file path is NULL");
  path_ = path;
  f_ = fopen(path, "rb");
  if (!f_) return io_fail("cannot open the state file", path_);
  struct stat sb{};
  if (fstat(fileno(f_), &sb) != 0) return io_fail("cannot stat the state file", path_);
  StateHeader hd{};
  if (fread(&hd, sizeof hd, 1, f_) != 1 || memcmp(hd.magic, kMagic, 8) != 0)
    return b2g_fail(B2G_EINVAL, "not a training-state file: " + path_);
  if (hd.version != kVersion) return b2g_fail(B2G_EINVAL, "unsupported training-state format version " + std::to_string(hd.version));
  if (hd.kind != kind)
    return b2g_fail(B2G_EINVAL, std::string("the state file belongs to a ") + (hd.kind == STATE_KIND_SAC ? "SAC" : hd.kind == STATE_KIND_BDQ ? "BDQ" : "unknown") +
                                    " learner");
  if (hd.n_fp != fp.size() || hd.n_sec > 64) return b2g_fail(B2G_EINVAL, "corrupt training-state header");
  std::vector<FpField> got(fp.size());
  if (!got.empty() && fread(got.data(), sizeof(FpField), got.size(), f_) != got.size())
    return b2g_fail(B2G_EINVAL, "truncated training-state header");
  for (size_t i = 0; i < fp.size(); ++i) {
    if (strncmp(got[i].name, fp[i].name, sizeof got[i].name) != 0 || got[i].kind != fp[i].kind)
      return b2g_fail(B2G_EINVAL, std::string("configuration fingerprint differs: the file has field '") +
                                      std::string(got[i].name, strnlen(got[i].name, sizeof got[i].name)) + "' where this handle has '" + fp[i].name + "'");
    if (got[i].v != fp[i].v)
      return b2g_fail(B2G_EINVAL, std::string("configuration fingerprint differs in '") + fp[i].name + "': " + fp_value(got[i]) +
                                      " in the file, " + fp_value(fp[i]) + " in this handle");
  }
  std::vector<SecEntry> tab(hd.n_sec);
  if (!tab.empty() && fread(tab.data(), sizeof(SecEntry), tab.size(), f_) != tab.size())
    return b2g_fail(B2G_EINVAL, "truncated training-state header");
  uint64_t off = sizeof(StateHeader) + fp.size() * sizeof(FpField) + tab.size() * sizeof(SecEntry);
  for (const SecEntry& e : tab) {
    if (e.offset != off) return b2g_fail(B2G_EINVAL, "corrupt training-state section table");
    off += e.bytes;
    tags_.push_back(e.tag); offs_.push_back(e.offset); lens_.push_back(e.bytes); sums_.push_back(e.checksum);
  }
  if (off != hd.file_bytes || (uint64_t)sb.st_size != hd.file_bytes)
    return b2g_fail(B2G_EINVAL, "training-state file is truncated or padded: " + std::to_string((uint64_t)sb.st_size) + " bytes, the header says " +
                                    std::to_string(hd.file_bytes));
  return 0;
}

int StateReader::read_host(int i, void* dst, size_t bytes) {
  StatePiece p;
  p.host = dst; p.bytes = bytes;
  return read_pieces(i, {p});
}

int StateReader::read_pieces(int i, const std::vector<StatePiece>& pieces) {
  size_t total = 0, largest = 0;
  for (const auto& p : pieces) { total += p.bytes; if (!p.host) largest = std::max(largest, p.bytes); }
  if (i < 0 || i >= n_sections() || total != lens_[i]) return b2g_fail(B2G_EINVAL, "training-state section length mismatch");
  if (fseeko(f_, (off_t)offs_[i], SEEK_SET) != 0) return io_fail("cannot seek in the state file", path_);
  Staging st;
  if (int rc = st.init(largest)) return rc;
  Hasher hs;
  size_t c = 0;       // chunks staged so far: buffer c & 1 is refilled once the copy of chunk c - 2 has finished
  for (const StatePiece& p : pieces) {
    if (p.host) {
      if (p.bytes && fread(p.host, 1, p.bytes, f_) != p.bytes) return io_fail("cannot read the state file", path_);
      hs.update(p.host, p.bytes);
      continue;
    }
    // the read of chunk k + 1 overlaps the host-to-device copy of chunk k
    for (size_t o = 0; o < p.bytes; o += st.chunk, ++c) {
      const size_t n = std::min(st.chunk, p.bytes - o);
      unsigned char* b = st.buf[c & 1];
      if (c >= 2) CK(cudaEventSynchronize(st.ev[c & 1]));
      if (fread(b, 1, n, f_) != n) return io_fail("cannot read the state file", path_);
      hs.update(b, n);
      CK(cudaMemcpyAsync((unsigned char*)p.dev + o, b, n, cudaMemcpyHostToDevice, st.s));
      CK(cudaEventRecord(st.ev[c & 1], st.s));
    }
  }
  if (st.s) CK(cudaStreamSynchronize(st.s));
  if (hs.digest() != sums_[i]) {
    const uint32_t t = tags_[i];
    const char tag[5] = {(char)(t & 255), (char)(t >> 8 & 255), (char)(t >> 16 & 255), (char)(t >> 24), 0};
    return b2g_fail(B2G_EINVAL, std::string("training-state section ") + tag + " fails its checksum");
  }
  return 0;
}

std::vector<StateSection> host_sections(void* host, size_t host_bytes, void* counters, size_t counter_bytes) {
  std::vector<StateSection> s(2);
  s[0].tag = state_tag("HOST"); s[0].pieces = {host_piece(host, host_bytes)};
  s[1].tag = state_tag("CNTR"); s[1].pieces = {host_piece(counters, counter_bytes)};
  return s;
}

std::vector<StateSection> adam_sections(float* P, size_t n_param, float* Mo, float* Vo, size_t n_moments) {
  std::vector<StateSection> s(3);
  s[0].tag = state_tag("PARM"); s[0].pieces = {dev_piece(P, n_param * sizeof(float))};
  s[1].tag = state_tag("ADMM"); s[1].pieces = {dev_piece(Mo, n_moments * sizeof(float))};
  s[2].tag = state_tag("ADMV"); s[2].pieces = {dev_piece(Vo, n_moments * sizeof(float))};
  return s;
}

int state_check_tags(const StateReader& rd, const std::vector<StateSection>& dev, const char* learner) {
  bool ok = rd.n_sections() == 2 + (int)dev.size() && rd.tag(0) == state_tag("HOST") && rd.tag(1) == state_tag("CNTR");
  for (int i = 0; ok && i < (int)dev.size(); ++i) ok = rd.tag(2 + i) == dev[i].tag;
  return ok ? 0 : b2g_fail(B2G_EINVAL, std::string("training-state file has the wrong sections for a ") + learner + " learner");
}

int state_check_lengths(const StateReader& rd, const std::vector<StateSection>& dev) {
  for (int i = 0; i < (int)dev.size(); ++i)
    if (rd.bytes(2 + i) != dev[i].bytes())
      return b2g_fail(B2G_EINVAL, "training-state section lengths do not match this handle's configuration");
  return 0;
}

int state_read_device(StateReader& rd, const std::vector<StateSection>& dev, bool* broken, const std::function<int()>& restore) {
  *broken = true;
  for (int i = 0; i < (int)dev.size(); ++i)
    if (int rc = rd.read_pieces(2 + i, dev[i].pieces)) return rc;
  if (int rc = restore()) return rc;
  *broken = false;
  return 0;
}

std::vector<FpField> fp_with_rms(std::vector<FpField> fp, bool owns_rms) {
  if (owns_rms) fp.push_back(fp_int("obs_rms", 1));
  return fp;
}

StateSection rms_section(double* count, double* mean, double* var, int E) {
  StateSection r;
  r.tag = state_tag("ORMS");
  r.pieces = {host_piece(count, sizeof(double)), dev_piece(mean, E * sizeof(double)), dev_piece(var, E * sizeof(double))};
  return r;
}

int state_fp_field(const char* path, uint32_t kind, const char* name) {
  FILE* f = path ? fopen(path, "rb") : nullptr;
  if (!f) return -1;
  StateHeader hd{};
  int found = -1;
  if (fread(&hd, sizeof hd, 1, f) == 1 && memcmp(hd.magic, kMagic, 8) == 0 && hd.kind == kind && hd.n_fp <= 64) {
    found = 0;
    FpField fp{};
    for (uint32_t i = 0; i < hd.n_fp && fread(&fp, sizeof fp, 1, f) == 1; ++i)
      if (strncmp(fp.name, name, sizeof fp.name) == 0) found = 1;
  }
  fclose(f);
  return found;
}

int state_open_rms(StateReader& rd, const char* path, uint32_t kind, const std::vector<FpField>& fp, bool owns_rms, const char* rms_set_call) {
  const int rc = rd.open(path, kind, fp_with_rms(fp, owns_rms));
  if (rc == 0) return 0;
  // a file with one fingerprint field more or fewer than this handle: say which side owns obs_rms
  const std::string msg = g_b2g_err;
  StateReader other;
  if (other.open(path, kind, fp_with_rms(fp, !owns_rms)) == 0)
    return b2g_fail(B2G_EINVAL, owns_rms ? std::string("the state file has no obs_rms, but this handle owns the observation statistics (") +
                                               rms_set_call + ")"
                                         : std::string("the state file carries obs_rms: call ") + rms_set_call + " on this handle before loading it");
  return b2g_fail(rc, msg);
}

}  // namespace b2g
