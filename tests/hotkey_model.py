"""A plain Python model of the hot-key collectors (incubator_pegasus_b200/host/hotkey.h, restating
src/server/hotkey_collector.cpp): the bucket hash of format.h, find_outlier_index and the collector's state machine with an
explicit clock.  The CPU tests check it against the golden cases, the GPU tests drive it next to the library."""
import math

M64 = (1 << 64) - 1
STOPPED, COARSE, FINE, FINISHED = 0, 1, 2, 3
START, STOP, QUERY = 0, 1, 2
OK, BUSY, INVALID_STATE, INVALID_PARAMETERS = 0, 1, 2, 3
QUEUE_CAP = 1000


def _mix(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def hotkey_hash(b: bytes) -> int:
    """format.h hotkey_hash: the sum of the mixed 32-bit words, finished with the length"""
    s = 0
    for j in range(0, (len(b) + 3) // 4):
        w = int.from_bytes(b[4 * j:4 * j + 4].ljust(4, b"\0"), "little")
        s = (s + _mix(((j << 32 | w) + 0x9E3779B97F4A7C15) & M64)) & M64
    return _mix(s ^ ((len(b) * 0xD6E8FEB86659FD93) & M64))


def bucket(hash_key: bytes, n_buckets: int) -> int:
    return hotkey_hash(hash_key) % n_buckets


def hash_key_of(raw_key: bytes) -> bytes:
    """format.h split_key: a hash-key length past the key is clamped to it"""
    if len(raw_key) < 2:
        return b""
    hkl = min(int.from_bytes(raw_key[:2], "big"), len(raw_key) - 2)
    return raw_key[2:2 + hkl]


def _to_int32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def find_outlier_index(values, threshold, hot_index=-1):
    """-> (found, hot_index), hot_index in / out as in the reference"""
    n = len(values)
    assert n > 2
    total = 0.0
    hot_value = 0
    for i, v in enumerate(values):
        total += v
        if v > (hot_value & M64):
            hot_index, hot_value = i, _to_int32(v)
    if hot_index == -1:
        return False, -1
    avg = (total - values[hot_index]) / (n - 1)
    sd = 0.0
    for i, v in enumerate(values):
        if i != hot_index:
            sd += (v - avg) ** 2
    sd = math.sqrt(sd / (n - 2))
    if sd == 0:
        return hot_value > avg, hot_index
    if (hot_value - avg) / sd >= threshold:
        return True, hot_index
    return False, -1


class Collector:
    def __init__(self, buckets=37, bucket_threshold=7, key_threshold=5, max_seconds=150):
        self.nb, self.bt, self.kt, self.max_s = buckets, bucket_threshold, key_threshold, max_seconds
        self._stop()

    def _stop(self):
        self.state, self.result, self.target, self.start_s = STOPPED, b"", -1, 0
        self.buckets = [0] * self.nb
        self.queue = []

    def control(self, action, now):
        if action == START:
            if self.state != STOPPED:
                return BUSY
            self.state, self.start_s = COARSE, now
            return OK
        if action == STOP:
            self._stop()
            return OK
        if action == QUERY:
            return OK if self.state == FINISHED else BUSY
        return INVALID_STATE

    def capture_raw_key(self, raw_key, weight=1):
        self.capture_hash_key(hash_key_of(raw_key), weight)

    def capture_hash_key(self, hk, weight=1):
        w = weight if weight > 0 else 1
        if self.state == COARSE:
            self.buckets[bucket(hk, self.nb)] += w
        elif self.state == FINE and bucket(hk, self.nb) == self.target and len(self.queue) < QUEUE_CAP:
            self.queue.append((hk, w))

    def analyse(self, now):
        if self.state not in (COARSE, FINE):
            return
        if now >= self.start_s + self.max_s:
            self._stop()
            return
        if self.state == COARSE:
            b, self.buckets = self.buckets, [0] * self.nb
            found, idx = find_outlier_index(b, self.bt, self.target)
            self.target = idx if found else -1
            if found:
                self.state = FINE
            return
        agg = {}
        for k, w in self.queue:
            agg[k] = agg.get(k, 0) + w
        self.queue = []
        if not agg:
            return
        keys = sorted(agg)  # heaviest-key ties go to the smallest key
        weights = [agg[k] for k in keys]
        best = max(weights)
        top = keys[weights.index(best)]
        if len(weights) < 3 or find_outlier_index(weights, self.kt, -1)[0]:
            self.result, self.state = top, FINISHED
