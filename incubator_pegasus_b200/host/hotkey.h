// hotkey.h — the hot-key collectors of one replica (src/server/hotkey_collector.{h,cpp}): the state machine, the coarse bucket
// counters and the fine queue of the host, and both analyses.  Plain C++ (no CUDA): the device side of the read collector
// (coarse counters in HBM, fine-queue tickets, hotkey_kernels.cuh) hands its captures over through device_phase() /
// add_fine_keys() and the bucket counts given to analyse().
//
//   START    STOPPED -> COARSE_DETECTING (OK); any other state: BUSY with a hint
//   STOP     any state -> STOPPED, counters and queue cleared (OK)
//   QUERY    FINISHED: OK with the hot hash key; any other state: BUSY with a hint
//   capture  COARSE: bucket hotkey_bucket(hash_key) += weight;  FINE: (hash_key, weight) queued when the key is in the target
//            bucket and the queue holds fewer than kHotkeyQueueCap entries.  A weight <= 0 counts as 1.
//   analyse  every hotkey_analyse_time_interval_s (the caller's timer): after max_seconds_to_detect_hotkey since START the
//            collector returns to STOPPED; otherwise COARSE reads and resets the buckets and moves to FINE when
//            find_outlier_index(buckets, hot_bucket_variance_threshold) finds a bucket, and FINE aggregates the queue by hash
//            key and moves to FINISHED when there are fewer than three distinct keys or find_outlier_index(weights,
//            hot_key_variance_threshold) finds one.  Heaviest-key ties go to the smallest key (the reference leaves them to
//            its hash map's order).
#pragma once
#include <atomic>
#include <cstdint>
#include <mutex>
#include <string>
#include <string_view>
#include <utility>
#include <vector>

namespace pgs {

enum HotkeyType : int32_t { HOTKEY_READ = 0, HOTKEY_WRITE = 1 };          // dsn::replication::hotkey_type
enum HotkeyAction : int32_t { HOTKEY_START = 0, HOTKEY_STOP = 1, HOTKEY_QUERY = 2 }; // dsn::replication::detect_action
enum HotkeyState : uint32_t { HOTKEY_STOPPED = 0, HOTKEY_COARSE = 1, HOTKEY_FINE = 2, HOTKEY_FINISHED = 3 };
// outcomes of a control request (the dsn error codes of detect_hotkey_response)
enum HotkeyOutcome : int32_t { HOTKEY_OK = 0, HOTKEY_BUSY = 1, HOTKEY_INVALID_STATE = 2, HOTKEY_INVALID_PARAMETERS = 3 };

constexpr uint32_t kHotkeyQueueCap = 1000; // hotkey_fine_data_collector's max_queue_size

struct HotkeyConfig {
    uint32_t buckets = 37;           // hotkey_buckets_num
    uint32_t bucket_threshold = 7;   // hot_bucket_variance_threshold
    uint32_t key_threshold = 5;      // hot_key_variance_threshold
    uint32_t max_seconds = 150;      // max_seconds_to_detect_hotkey
};
// the knobs as pgs_server_options carries them: 0 = the default; false when the bucket count is not a prime >= 3
bool hotkey_config(uint32_t buckets, uint32_t bucket_threshold, uint32_t key_threshold, uint32_t max_seconds, HotkeyConfig &out);

// hotkey_collector.cpp:82-128, restated: the 68-95-99.7 rule over all values but the largest.  hot_index is in / out as in
// the reference (it is only written when a value above 0 is seen, and reset to -1 when the largest is not an outlier).
// Requires values.size() > 2.
bool find_outlier_index(const std::vector<uint64_t> &values, int threshold, int &hot_index);

const char *hotkey_state_name(uint32_t state);

class HotkeyCollector {
public:
    explicit HotkeyCollector(HotkeyType type) : type_(type) { set_config(HotkeyConfig{}); }
    void set_config(const HotkeyConfig &c);
    const HotkeyConfig &config() const { return cfg_; }
    HotkeyType type() const { return type_; }
    uint32_t state() const { return state_.load(std::memory_order_acquire); }
    bool active() const { uint32_t s = state(); return s == HOTKEY_COARSE || s == HOTKEY_FINE; }

    // capture_raw_key / capture_hash_key
    void capture_raw_key(std::string_view raw_key, int64_t weight);
    void capture_hash_key(std::string_view hash_key, int64_t weight);

    // START / STOP / QUERY at `now` (seconds).  text = the hint, or the hot hash key of a successful QUERY.
    int32_t control(int32_t action, uint32_t now, std::string &text);
    // one analysis step at `now`.  device_buckets: coarse counts captured elsewhere since the last step (the device's), added
    // to the host's own before the analysis; null or empty = none.
    void analyse(uint32_t now, const std::vector<uint64_t> *device_buckets = nullptr);

    // device capture: the phase a launch captures in, and the queue room it may fill (0 outside FINE)
    struct Phase { uint32_t state; uint32_t target; uint32_t room; };
    Phase device_phase() const;
    // fine-phase keys captured elsewhere (weight 1 each), appended while the queue has room
    void add_fine_keys(const std::vector<std::string> &hash_keys);

    // inspection (tests)
    std::string result() const;
    int32_t target_bucket() const;
    size_t queue_size() const;
    std::vector<uint64_t> buckets() const;

private:
    void stop_locked();
    bool push_locked(std::string_view hash_key, uint64_t weight);
    HotkeyType type_;
    HotkeyConfig cfg_;
    mutable std::mutex mu_;
    std::atomic<uint32_t> state_{HOTKEY_STOPPED};
    uint32_t start_s_ = 0;
    int32_t target_ = -1;
    std::string result_;
    std::vector<uint64_t> buckets_;
    std::vector<std::pair<std::string, uint64_t>> queue_;
};

} // namespace pgs
