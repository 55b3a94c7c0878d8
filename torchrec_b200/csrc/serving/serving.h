// Native core of the inference server: request intake, dynamic batching into pinned staging buffers, per-GPU ready
// queues with back-pressure, and result splitting back to per-request futures.
//
// Parity: reference torchrec/inference(_legacy): BatchingQueue (BatchingQueue.h/.cpp), Batching.cpp (dense / sparse
// combine), GPUExecutor + ResourceManager (outstanding-batch limits), ResultSplit.cpp, Observer.h. Re-designed around
// GPU serving: the batcher writes ONE contiguous pinned slab per batch (dense | lengths | values | weights...) so the
// executor issues a single H2D copy per batch, and sparse features are merged straight into the key-major KJT layout the
// embedding kernels consume (no per-feature tensors, no second permute on the device).
#pragma once
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

namespace trbs {

using Clock = std::chrono::steady_clock;

struct SparseInput {
  int32_t num_features = 0;
  std::vector<int32_t> lengths;  // [num_features * batch]
  std::vector<int64_t> values;   // jagged, key-major
  std::vector<float> weights;    // empty or same length as values
};

struct Request {
  int64_t id = 0;
  int32_t batch_size = 0;
  int32_t num_float = 0;
  std::vector<float> dense;  // [batch, num_float]
  SparseInput id_list;
  SparseInput id_score_list;
  Clock::time_point enqueued;
  // result
  std::mutex mu;
  std::condition_variable cv;
  bool done = false;
  int status = 0;
  std::vector<float> result;  // [batch, outputs_per_sample]
};

// Layout of one formed batch inside its slab (byte offsets, -1 = absent)
struct BatchDesc {
  int64_t batch_id;
  int32_t buffer_index;
  int32_t batch_size;
  int32_t num_requests;
  int32_t num_float;
  int32_t id_list_features;
  int32_t id_score_features;
  int64_t dense_off;
  int64_t idl_lengths_off, idl_values_off, idl_num_values;
  int64_t ids_lengths_off, ids_values_off, ids_weights_off, ids_num_values;
  int64_t total_bytes;
  int64_t oldest_wait_us;  // queueing delay of the oldest request when the batch was formed
};

struct Stats {
  std::atomic<int64_t> requests{0}, batches{0}, samples{0}, rejected{0}, timeouts{0};
  std::atomic<int64_t> queue_us_sum{0}, queue_us_max{0}, exec_us_sum{0};
};

struct Config {
  int32_t max_batch_size = 2048;
  int64_t batching_interval_us = 1000;
  int32_t num_gpus = 1;
  int32_t max_outstanding_per_gpu = 2;
  int32_t batching_threads = 2;
  int64_t max_queue_requests = 1 << 16;
};

class Server {
 public:
  explicit Server(const Config& cfg);
  ~Server();
  void add_buffer(void* ptr, int64_t bytes);  // pinned staging slab (owned by the caller)
  // returns request id, or -1 when the intake queue is full
  int64_t submit(int32_t batch_size, int32_t num_float, const float* dense, int32_t idl_features, const int32_t* idl_lengths, const int64_t* idl_values,
                 int64_t idl_nvalues, int32_t ids_features, const int32_t* ids_lengths, const int64_t* ids_values, const float* ids_weights, int64_t ids_nvalues);
  // executor side
  int pop_batch(int gpu, int64_t timeout_us, BatchDesc* out);  // 0 ok, 1 timeout, 2 shutting down
  int complete(int64_t batch_id, const float* preds, int32_t outputs_per_sample, int status);
  // client side: 0 ok, 1 timeout, <0 error status. *n_out receives the number of floats written
  int wait(int64_t request_id, float* out, int64_t max_floats, int64_t timeout_us, int64_t* n_out);
  void shutdown();
  const Stats& stats() const { return stats_; }

 private:
  struct Formed {
    BatchDesc desc;
    std::vector<std::shared_ptr<Request>> requests;
    Clock::time_point formed_at;
    int gpu;
  };
  void batching_loop();
  bool form_batch(std::vector<std::shared_ptr<Request>>& reqs);
  int acquire_buffer(int64_t bytes, uint8_t** ptr);

  Config cfg_;
  Stats stats_;
  std::atomic<bool> stop_{false};
  std::atomic<int64_t> next_request_{1}, next_batch_{1};
  // intake
  std::mutex in_mu_;
  std::condition_variable in_cv_;
  std::deque<std::shared_ptr<Request>> intake_;
  std::map<int64_t, std::shared_ptr<Request>> live_;  // request id -> request (until waited)
  // buffers
  struct Buffer { uint8_t* ptr; int64_t bytes; bool busy; };
  std::mutex buf_mu_;
  std::condition_variable buf_cv_;
  std::vector<Buffer> buffers_;
  // ready queues + in-flight accounting per gpu
  std::mutex rq_mu_;
  std::condition_variable rq_cv_;
  std::vector<std::deque<std::shared_ptr<Formed>>> ready_;
  std::vector<int> outstanding_;
  std::map<int64_t, std::shared_ptr<Formed>> inflight_;
  int rr_ = 0;
  std::vector<std::thread> threads_;
};

}  // namespace trbs
