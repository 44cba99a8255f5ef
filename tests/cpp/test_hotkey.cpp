// The hot-key collectors' host logic (incubator_pegasus_b200/host/hotkey.h) against the reference's own unit tests
// (src/server/test/hotkey_collector_test.cpp): the find_outlier_index cases of a fixture file (argv[1], written from
// tests/golden/hotkey_outliers.json by tests/test_hotkey_host.py), the state transitions of :303-368 and the fine collector
// of :187-227, driven with an explicit clock, plus the 150 s timeout and the cap of 1000 queued captures.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <random>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "../../incubator_pegasus_b200/csrc/format.h"
#include "../../incubator_pegasus_b200/host/hotkey.cpp"

using namespace pgs;

#define CHECK(c)                                                                  \
    do {                                                                          \
        if (!(c)) { fprintf(stderr, "%s:%d: CHECK(%s) failed\n", __FILE__, __LINE__, #c); exit(1); } \
    } while (0)

static const std::string kHot = "ThisisahotkeyThisisahotkey";
static std::mt19937 rng(7);

// generate_hash_key_by_random (hotkey_collector_test.cpp:38-70): the hot key with probability `probability` percent
static std::string random_hash_key(bool is_hotkey, int probability = 100)
{
    if (is_hotkey && (int)(rng() % 100) < probability) return kHot;
    static const std::string chars = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ1234567890!@#$%^&*()`~-_=+[{]{\\|;:'\",<.>/? ";
    std::string r;
    for (int i = 0; i < 20; i++) r += chars[rng() % chars.size()];
    return r;
}
static std::string raw_key(const std::string &hk, const std::string &sk)
{
    std::string k(2, '\0');
    k[0] = (char)(hk.size() >> 8); k[1] = (char)hk.size();
    return k + hk + sk;
}

static void outlier_cases(const char *path)
{
    std::ifstream f(path);
    CHECK(f.good());
    std::string line;
    int n_cases = 0;
    while (std::getline(f, line)) {
        std::istringstream in(line);
        int threshold, found, index;
        size_t n;
        in >> threshold >> found >> index >> n;
        std::vector<uint64_t> v(n);
        for (auto &x : v) in >> x;
        int hot = -1;
        const bool got = find_outlier_index(v, threshold, hot);
        if (got != (found != 0) || hot != index) { fprintf(stderr, "case %d: found %d index %d, expected %d %d\n", n_cases, got, hot, found, index); exit(1); }
        n_cases++;
    }
    CHECK(n_cases >= 4);
    printf("outlier cases: %d\n", n_cases);
}

static void state_transform()
{
    HotkeyCollector c(HOTKEY_READ);
    std::string text;
    uint32_t now = 1000;
    CHECK(c.state() == HOTKEY_STOPPED);
    CHECK(c.control(HOTKEY_QUERY, now, text) == HOTKEY_BUSY);
    CHECK(c.control(HOTKEY_START, now, text) == HOTKEY_OK && c.state() == HOTKEY_COARSE);
    CHECK(c.control(HOTKEY_START, now, text) == HOTKEY_BUSY && c.state() == HOTKEY_COARSE);
    // captures from several handler threads, as the reference's tasks do
    std::vector<std::thread> ts;
    for (int t = 0; t < 4; t++) {
        std::vector<std::string> keys;
        for (int i = 0; i < 25; i++) keys.push_back(raw_key(random_hash_key(true, 80), "sortkey"));
        ts.emplace_back([&c, keys] { for (auto &k : keys) c.capture_raw_key(k, 1); });
    }
    for (auto &t : ts) t.join();
    c.analyse(now += 10);
    CHECK(c.state() == HOTKEY_FINE);
    for (int i = 0; i < 100; i++) c.capture_raw_key(raw_key(random_hash_key(true, 80), "sortkey"), 1);
    c.analyse(now += 10);
    CHECK(c.state() == HOTKEY_FINISHED);
    CHECK(c.result() == kHot);
    CHECK(c.control(HOTKEY_QUERY, now, text) == HOTKEY_OK && text == kHot);
    CHECK(c.control(HOTKEY_START, now, text) == HOTKEY_BUSY && c.state() == HOTKEY_FINISHED);
    CHECK(c.control(HOTKEY_STOP, now, text) == HOTKEY_OK && c.state() == HOTKEY_STOPPED && c.result().empty());
    CHECK(c.control(HOTKEY_START, now, text) == HOTKEY_OK && c.state() == HOTKEY_COARSE);
    for (int i = 0; i < 1000; i++) c.capture_raw_key(raw_key(random_hash_key(false), "sortkey"), 1);
    c.analyse(now += 10);
    CHECK(c.state() == HOTKEY_COARSE);
    CHECK(c.control(HOTKEY_STOP, now, text) == HOTKEY_OK && c.state() == HOTKEY_STOPPED);
    CHECK(c.control(7, now, text) == HOTKEY_INVALID_STATE);
}

static void timeout()
{
    HotkeyCollector c(HOTKEY_WRITE);
    std::string text;
    const uint32_t t0 = 5000;
    CHECK(c.control(HOTKEY_START, t0, text) == HOTKEY_OK);
    for (uint32_t t = t0 + 10; t < t0 + 150; t += 10) {
        for (int i = 0; i < 1000; i++) c.capture_hash_key(random_hash_key(false), 1);
        c.analyse(t);
        CHECK(c.state() == HOTKEY_COARSE);
    }
    c.analyse(t0 + 150);
    CHECK(c.state() == HOTKEY_STOPPED);
    // the timeout holds in the fine phase too
    CHECK(c.control(HOTKEY_START, t0 + 200, text) == HOTKEY_OK);
    for (int i = 0; i < 200; i++) c.capture_hash_key(kHot, 1);
    c.analyse(t0 + 210);
    CHECK(c.state() == HOTKEY_FINE);
    c.analyse(t0 + 349);
    CHECK(c.state() == HOTKEY_FINE); // an empty queue finds nothing
    c.analyse(t0 + 350);
    CHECK(c.state() == HOTKEY_STOPPED);
}

// keys of the target bucket only, as the reference's fine collector of one bucket sees them
static std::string in_bucket(const HotkeyCollector &c, bool is_hotkey, int probability = 100)
{
    for (;;) {
        std::string k = random_hash_key(is_hotkey, probability);
        if ((int32_t)hotkey_bucket((const uint8_t *)k.data(), (uint32_t)k.size(), c.config().buckets) == c.target_bucket()) return k;
    }
}

static void fine_collector()
{
    HotkeyCollector c(HOTKEY_READ);
    std::string text;
    uint32_t now = 100;
    CHECK(c.control(HOTKEY_START, now, text) == HOTKEY_OK);
    for (int i = 0; i < 300; i++) c.capture_hash_key(kHot, 1);
    c.analyse(now += 10);
    CHECK(c.state() == HOTKEY_FINE);
    CHECK(c.target_bucket() == (int32_t)hotkey_bucket((const uint8_t *)kHot.data(), (uint32_t)kHot.size(), 37));
    for (int i = 0; i < 1000; i++) c.capture_hash_key(in_bucket(c, true, 80), 1);
    CHECK(c.queue_size() == 1000);
    // a fresh fine period with uniform keys finds nothing, and the queue never holds more than 1000 entries
    HotkeyCollector d(HOTKEY_READ);
    CHECK(d.control(HOTKEY_START, now, text) == HOTKEY_OK);
    for (int i = 0; i < 300; i++) d.capture_hash_key(kHot, 1);
    d.analyse(now + 10);
    CHECK(d.state() == HOTKEY_FINE);
    for (int i = 0; i < 1000; i++) d.capture_hash_key(in_bucket(d, false), 1);
    d.analyse(now + 20);
    CHECK(d.state() == HOTKEY_FINE && d.result().empty() && d.queue_size() == 0);
    for (int i = 0; i < 5000; i++) d.capture_hash_key(in_bucket(d, true, 80), 1);
    CHECK(d.queue_size() == kHotkeyQueueCap);
    // keys outside the target bucket are not queued
    std::string other;
    do other = random_hash_key(false); while ((int32_t)hotkey_bucket((const uint8_t *)other.data(), (uint32_t)other.size(), 37) == d.target_bucket());
    d.analyse(now + 30);
    CHECK(d.state() == HOTKEY_FINISHED && d.result() == kHot);
    c.analyse(now += 10);
    CHECK(c.state() == HOTKEY_FINISHED && c.result() == kHot);
    CHECK(c.control(HOTKEY_STOP, now, text) == HOTKEY_OK && c.queue_size() == 0);
    HotkeyCollector e(HOTKEY_READ);
    CHECK(e.control(HOTKEY_START, now, text) == HOTKEY_OK);
    for (int i = 0; i < 300; i++) e.capture_hash_key(kHot, 1);
    e.analyse(now + 10);
    e.capture_hash_key(other, 1);
    CHECK(e.queue_size() == 0);
    // device hand-over: the room shrinks as the queue fills, and keys past the cap are dropped
    CHECK(e.device_phase().state == HOTKEY_FINE && e.device_phase().room == kHotkeyQueueCap);
    e.add_fine_keys(std::vector<std::string>(600, kHot));
    CHECK(e.device_phase().room == kHotkeyQueueCap - 600);
    e.add_fine_keys(std::vector<std::string>(600, kHot));
    CHECK(e.queue_size() == kHotkeyQueueCap && e.device_phase().room == 0);
}

static void weights_and_config()
{
    HotkeyConfig cfg;
    CHECK(hotkey_config(0, 0, 0, 0, cfg) && cfg.buckets == 37 && cfg.bucket_threshold == 7 && cfg.key_threshold == 5 && cfg.max_seconds == 150);
    CHECK(!hotkey_config(1, 0, 0, 0, cfg) && !hotkey_config(2, 0, 0, 0, cfg) && !hotkey_config(39, 0, 0, 0, cfg) && !hotkey_config(49, 0, 0, 0, cfg));
    CHECK(hotkey_config(3, 0, 0, 0, cfg) && hotkey_config(101, 1, 2, 3, cfg) && cfg.buckets == 101 && cfg.max_seconds == 3);
    HotkeyCollector c(HOTKEY_WRITE);
    std::string text;
    c.capture_hash_key("x", 5); // stopped: nothing
    CHECK(c.control(HOTKEY_START, 0, text) == HOTKEY_OK);
    c.capture_hash_key("x", 5);
    c.capture_hash_key("x", 0);  // a weight <= 0 counts as 1
    c.capture_hash_key("x", -3);
    c.capture_raw_key(std::string("\x00\x01xsort", 7), 1);
    const uint32_t b = hotkey_bucket((const uint8_t *)"x", 1, 37);
    uint64_t sum = 0;
    for (uint64_t v : c.buckets()) sum += v;
    CHECK(c.buckets()[b] == 8 && sum == 8);
}

int main(int argc, char **argv)
{
    if (argc < 2) { fprintf(stderr, "usage: test_hotkey cases.txt\n"); return 2; }
    outlier_cases(argv[1]);
    state_transform();
    timeout();
    fine_collector();
    weights_and_config();
    printf("OK\n");
    return 0;
}
