"""The job mixes of the multi-job compaction tests (pgs_compact_many), shared by the kernel simulator
(test_compact_many_sim.py) and the device (test_compact_many_gpu.py).  A job is a dict: runs (Records, the oldest first),
bottommost, kw (the filter keyword arguments of Partition.compact, with ops_json for an ops table)."""
import numpy as np

import merge_inputs
from incubator_pegasus_b200 import Records, synth

OPS_DELETE = (
    '{"ops":[{"type":"COT_DELETE","params":"","rules":[{"type":"FRT_SORTKEY_PATTERN","params":'
    '"{\\"pattern\\":\\"5\\",\\"match_type\\":\\"SMT_MATCH_POSTFIX\\"}"}]}]}'
)
OPS_TTL = (
    '{"ops":[{"type":"COT_UPDATE_TTL","params":"{\\"type\\":\\"UTOT_FROM_NOW\\",\\"value\\":500}","rules":['
    '{"type":"FRT_SORTKEY_PATTERN","params":"{\\"pattern\\":\\"3\\",\\"match_type\\":\\"SMT_MATCH_POSTFIX\\"}"}]}]}'
)


def tombstones_only(seed, n=60):
    """one run of deletions only: merged at the bottommost level nothing survives"""
    r = synth.compaction_runs(k=1, n_per_run=n, seed=seed)[0]
    return Records(r.keys, r.key_off, np.zeros(0, np.uint8), np.zeros(n + 1, np.uint64), r.seq,
                   np.full(n, synth.TYPE_DELETION, np.uint8))


def job(runs, bottommost, **kw):
    return dict(runs=runs, bottommost=bottommost, kw=kw)


def mix_main(scale=1):
    """different pidx / partition_version with validate_hash, different default_ttl and ops tables, bottommost 0 and 1, a
    one-run job, a 16-run job and a job whose output is empty"""
    return [
        job(synth.compaction_runs(k=3, n_per_run=150 * scale, sortkeys_per_hash=8, seed=11), True,
            validate_hash=True, pidx=1, partition_version=3),
        job(synth.compaction_runs(k=2, n_per_run=120 * scale, sortkeys_per_hash=16, seed=12), False,
            default_ttl=3600, ops_json=OPS_DELETE),
        job(synth.compaction_runs(k=1, n_per_run=100 * scale, seed=13), True,
            validate_hash=True, pidx=2, partition_version=3, default_ttl=60),
        job(synth.compaction_runs(k=16, n_per_run=20 * scale, sortkeys_per_hash=4, seed=14), False, ops_json=OPS_TTL),
        job([tombstones_only(15)], True),
    ]


def mix_long_keys():
    """a job of 2 KB user keys widens the key rows of every job of the launch"""
    return [
        job(synth.compaction_runs(k=3, n_per_run=100, sortkeys_per_hash=8, seed=21), True, validate_hash=True, pidx=0,
            partition_version=1),
        job(merge_inputs.long_keys(22), True, default_ttl=100),
        job(synth.compaction_runs(k=1, n_per_run=80, seed=23), False, ops_json=OPS_DELETE),
    ]


def mix_too_wide():
    """a 16-run job and a job of 2 KB keys: the deepest job's cursor states and the widest key's rows do not fit one launch"""
    return [job(synth.compaction_runs(k=16, n_per_run=20, seed=31), True), job(merge_inputs.long_keys(32), True)]
