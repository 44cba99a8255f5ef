// hotkey.cpp — the hot-key collectors' host logic (see hotkey.h).
#include "hotkey.h"

#include <cmath>
#include <map>

#include "../csrc/format.h"

namespace pgs {

bool hotkey_config(uint32_t buckets, uint32_t bucket_threshold, uint32_t key_threshold, uint32_t max_seconds, HotkeyConfig &out)
{
    HotkeyConfig c;
    if (buckets) c.buckets = buckets;
    if (bucket_threshold) c.bucket_threshold = bucket_threshold;
    if (key_threshold) c.key_threshold = key_threshold;
    if (max_seconds) c.max_seconds = max_seconds;
    if (c.buckets < 3) return false; // the flag validator of hotkey_buckets_num: a prime >= 3
    for (uint32_t i = 2; i <= c.buckets / i; i++)
        if (c.buckets % i == 0) return false;
    out = c;
    return true;
}

bool find_outlier_index(const std::vector<uint64_t> &values, int threshold, int &hot_index)
{
    const int data_size = (int)values.size();
    if (data_size <= 2) return false; // the reference CHECKs
    double sum = 0;
    int hot_value = 0; // an int, as in the reference
    for (int i = 0; i < data_size; i++) {
        sum += values[i];
        if (values[i] > (uint64_t)(int64_t)hot_value) {
            hot_index = i;
            hot_value = (int)values[i];
        }
    }
    if (hot_index == -1) return false;
    const double avg = (sum - values[hot_index]) / (data_size - 1);
    double sd = 0;
    for (int i = 0; i < data_size; i++)
        if (i != hot_index) sd += std::pow(values[i] - avg, 2);
    sd = std::sqrt(sd / (data_size - 2));
    // all values but the largest are equal ([1, 1, 300, 1] or [1, 1, 1, 1]): the largest is hot when it is above them
    if (sd == 0) return hot_value > avg;
    const double hot_point = (hot_value - avg) / sd;
    if (hot_point >= threshold) return true;
    hot_index = -1;
    return false;
}

const char *hotkey_state_name(uint32_t state)
{
    switch (state) {
    case HOTKEY_STOPPED: return "STOPPED";
    case HOTKEY_COARSE: return "COARSE_DETECTING";
    case HOTKEY_FINE: return "FINE_DETECTING";
    case HOTKEY_FINISHED: return "FINISHED";
    }
    return "UNKNOWN";
}

static const char *type_name(HotkeyType t) { return t == HOTKEY_READ ? "READ" : "WRITE"; }

void HotkeyCollector::set_config(const HotkeyConfig &c)
{
    std::lock_guard<std::mutex> g(mu_);
    cfg_ = c;
    stop_locked();
}

void HotkeyCollector::stop_locked()
{
    state_.store(HOTKEY_STOPPED, std::memory_order_release);
    result_.clear();
    target_ = -1;
    buckets_.assign(cfg_.buckets, 0);
    queue_.clear();
}

bool HotkeyCollector::push_locked(std::string_view hash_key, uint64_t weight)
{
    if (queue_.size() >= kHotkeyQueueCap) return false; // no room: the capture is dropped
    queue_.emplace_back(std::string(hash_key), weight);
    return true;
}

void HotkeyCollector::capture_raw_key(std::string_view raw_key, int64_t weight)
{
    if (!active()) return;
    const KeyParts k = split_key((const uint8_t *)raw_key.data(), (uint32_t)raw_key.size());
    capture_hash_key(std::string_view((const char *)k.hk, k.hkl), weight);
}

void HotkeyCollector::capture_hash_key(std::string_view hash_key, int64_t weight)
{
    if (!active()) return;
    const uint64_t w = weight > 0 ? (uint64_t)weight : 1u;
    const uint32_t b = hotkey_bucket((const uint8_t *)hash_key.data(), (uint32_t)hash_key.size(), cfg_.buckets);
    std::lock_guard<std::mutex> g(mu_);
    const uint32_t s = state();
    if (s == HOTKEY_COARSE) buckets_[b] += w;
    else if (s == HOTKEY_FINE && (int32_t)b == target_) push_locked(hash_key, w);
}

int32_t HotkeyCollector::control(int32_t action, uint32_t now, std::string &text)
{
    std::lock_guard<std::mutex> g(mu_);
    const uint32_t s = state();
    switch (action) {
    case HOTKEY_START:
        if (s == HOTKEY_COARSE || s == HOTKEY_FINE) {
            text = std::string("still detecting ") + type_name(type_) + " hotkey, state is " + hotkey_state_name(s);
            return HOTKEY_BUSY;
        }
        if (s == HOTKEY_FINISHED) {
            text = std::string(type_name(type_)) + " hotkey result has been found: " + result_ +
                   ", you can send a stop rpc to restart hotkey detection";
            return HOTKEY_BUSY;
        }
        start_s_ = now;
        state_.store(HOTKEY_COARSE, std::memory_order_release);
        text = std::string("starting to detect ") + type_name(type_) + " hotkey";
        return HOTKEY_OK;
    case HOTKEY_STOP:
        stop_locked();
        text = std::string(type_name(type_)) + " hotkey stopped, cache cleared";
        return HOTKEY_OK;
    case HOTKEY_QUERY:
        if (s != HOTKEY_FINISHED) {
            text = std::string("Can't get hotkey now, now state: ") + hotkey_state_name(s);
            return HOTKEY_BUSY;
        }
        text = result_;
        return HOTKEY_OK;
    }
    text = std::to_string(action) + ": can't find this detect action";
    return HOTKEY_INVALID_STATE;
}

void HotkeyCollector::analyse(uint32_t now, const std::vector<uint64_t> *device_buckets)
{
    std::lock_guard<std::mutex> g(mu_);
    const uint32_t s = state();
    if (s != HOTKEY_COARSE && s != HOTKEY_FINE) return;
    if ((uint64_t)now >= (uint64_t)start_s_ + cfg_.max_seconds) { // terminate_if_timeout
        stop_locked();
        return;
    }
    if (s == HOTKEY_COARSE) {
        std::vector<uint64_t> b(cfg_.buckets, 0);
        b.swap(buckets_);
        if (device_buckets)
            for (size_t i = 0; i < device_buckets->size() && i < b.size(); i++) b[i] += (*device_buckets)[i];
        int idx = target_;
        if (!find_outlier_index(b, (int)cfg_.bucket_threshold, idx)) idx = -1;
        target_ = idx;
        if (idx != -1) state_.store(HOTKEY_FINE, std::memory_order_release);
        return;
    }
    // FINE: aggregate the queue (at most one period's worth) by hash key
    std::map<std::string, uint64_t> weight;
    for (auto &e : queue_) weight[e.first] += e.second;
    queue_.clear();
    if (weight.empty()) return;
    std::vector<uint64_t> w;
    w.reserve(weight.size());
    const std::string *max_key = nullptr;
    uint64_t max_w = 0;
    for (auto &e : weight) {
        w.push_back(e.second);
        if (e.second > max_w) { max_w = e.second; max_key = &e.first; }
    }
    int hot_index = -1;
    if (w.size() < 3 || find_outlier_index(w, (int)cfg_.key_threshold, hot_index)) {
        result_ = *max_key;
        state_.store(HOTKEY_FINISHED, std::memory_order_release);
    }
}

HotkeyCollector::Phase HotkeyCollector::device_phase() const
{
    std::lock_guard<std::mutex> g(mu_);
    const uint32_t s = state();
    if (s == HOTKEY_FINE) return Phase{s, (uint32_t)target_, (uint32_t)(kHotkeyQueueCap - queue_.size())};
    return Phase{s == HOTKEY_COARSE ? s : (uint32_t)HOTKEY_STOPPED, 0, 0};
}

void HotkeyCollector::add_fine_keys(const std::vector<std::string> &hash_keys)
{
    std::lock_guard<std::mutex> g(mu_);
    if (state() != HOTKEY_FINE) return;
    for (auto &k : hash_keys)
        if (!push_locked(k, 1)) break;
}

std::string HotkeyCollector::result() const { std::lock_guard<std::mutex> g(mu_); return result_; }
int32_t HotkeyCollector::target_bucket() const { std::lock_guard<std::mutex> g(mu_); return target_; }
size_t HotkeyCollector::queue_size() const { std::lock_guard<std::mutex> g(mu_); return queue_.size(); }
std::vector<uint64_t> HotkeyCollector::buckets() const { std::lock_guard<std::mutex> g(mu_); return buckets_; }

} // namespace pgs
