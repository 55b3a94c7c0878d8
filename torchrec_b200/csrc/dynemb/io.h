// Parameter-server IO layer of the dynamic embedding runtime.
//
// An IO backend stores rows (opaque byte blobs) keyed by (table, column-group, global id). Backends are looked up by
// URL scheme in a process-wide registry: built in are `memory://<name>` (shared in-process store: the DDR tier of a
// HBM cache, and the test double) and `file://<dir>` (append-only log + in-memory index, survives restarts).
// External plugins (`.so` exporting `trb_io_plugin`) can be loaded at runtime, mirroring the reference's redis plugin
// (torchrec/csrc/dynamic_embedding/details/io_registry.h, io.h, redis/).
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <vector>

namespace trb {

class IOBackend {
 public:
  virtual ~IOBackend() = default;
  // rows: n consecutive blobs of row_bytes each
  virtual void push(const std::string& table, const int64_t* gids, int64_t n, const uint8_t* rows, int64_t row_bytes) = 0;
  // found[i] = 1 when gid i exists (its blob is copied to rows + i*row_bytes), else 0 and the blob is left untouched
  virtual void pull(const std::string& table, const int64_t* gids, int64_t n, uint8_t* rows, int64_t row_bytes, uint8_t* found) = 0;
  virtual int64_t size(const std::string& table) = 0;
};

// C plugin ABI (all functions required)
struct IOPlugin {
  void* (*create)(const char* url);
  void (*destroy)(void* self);
  void (*push)(void* self, const char* table, const int64_t* gids, int64_t n, const uint8_t* rows, int64_t row_bytes);
  void (*pull)(void* self, const char* table, const int64_t* gids, int64_t n, uint8_t* rows, int64_t row_bytes, uint8_t* found);
  int64_t (*size)(void* self, const char* table);
};

using IOFactory = std::function<std::shared_ptr<IOBackend>(const std::string& url)>;

class IORegistry {
 public:
  static IORegistry& instance();
  void add(const std::string& scheme, IOFactory f);
  bool load_plugin(const std::string& scheme, const std::string& so_path);  // dlopen + `trb_io_plugin`
  std::shared_ptr<IOBackend> open(const std::string& url);

 private:
  IORegistry();
  struct Impl;
  std::shared_ptr<Impl> impl_;
};

}  // namespace trb
