"""TEST INFRASTRUCTURE — the oracle's outputs on the stand-in asset pack, recorded once and replayed.

An `oracle_env` is, while recording (PG_ORACLE_RECORD_DIR set, oracle/_ref built), the oracle itself; otherwise
it is the library under test behind the same libenv ABI. Either way every observation (rew, rgb, first, info)
and every state blob it returns is folded into a running sha256, and the digest after every EVERY-th output
and after the last one is written (recording) or must equal what the oracle wrote (tests/golden/
oracle_records.json.gz). A test that compares the library with an `oracle_env` therefore compares it with the
oracle's recorded outputs, on any machine. Records are keyed by the test's file and name (test_key; or an
explicit key) and the order in which the test creates its oracle envs.
"""
from __future__ import annotations

import gzip
import hashlib
import json
import os
import re

import numpy as np

from oracle.ref_env import REF_LIB, RefVecEnv

HERE = os.path.dirname(os.path.abspath(__file__))
RECORDS = os.path.join(os.path.dirname(HERE), "tests", "golden", "oracle_records.json.gz")
STANDIN_PACK = os.path.join(os.path.dirname(HERE), "procgen_b200", "data", "standin.pack")
EVERY = 200
_records = None
_counters = {}


def recording_dir():
    return os.environ.get("PG_ORACLE_RECORD_DIR") or None


def test_key(nodeid):
    """The test file's name and the test's name: pytest's node id without the directories, which depend on
    the rootdir pytest picked for the run."""
    nodeid = re.sub(r" \((setup|call|teardown)\)$", "", nodeid)
    path, sep, name = nodeid.partition("::")
    return os.path.basename(path) + sep + name


def _next_key(key=None):
    """The record of the next oracle env: `key` as given when it names one env ("<test key>#<n>", which is how
    a test replays another test's record), else the test's key numbered by the envs it created so far."""
    if key and "#" in key:
        return key
    base = key or test_key(os.environ.get("PYTEST_CURRENT_TEST", "unkeyed"))
    k = _counters.get(base, 0)
    _counters[base] = k + 1
    return f"{base}#{k}"


def _load():
    global _records
    if _records is None:
        with gzip.open(RECORDS, "rt") as f:
            _records = json.load(f)
    return _records


def use_records(path):
    """Make the records of another record file (e.g. tests/golden/level_seed_records.json.gz) replayable through
    oracle_env beside those of RECORDS. A file of its own keeps a new test file's records apart from the
    existing ones; its keys are its tests' own, and a key in both files must hold the same digests."""
    if recording_dir():
        return
    recs = _load()
    with gzip.open(path, "rt") as f:
        extra = json.load(f)
    clash = [k for k in extra if k in recs and recs[k] != extra[k]]
    assert not clash, f"records in {os.path.basename(path)} and {os.path.basename(RECORDS)} differ: {clash[:4]}"
    recs.update(extra)


class Checked:
    """An env of the libenv ABI (RefVecEnv) whose outputs are checked against, or recorded as, the oracle's."""

    def __init__(self, env, key):
        self.env, self.key = env, key
        self.h = hashlib.sha256()
        self.n = 0
        self.marks = []
        self.want = None if recording_dir() else _load().get(key)
        if self.want is None and not recording_dir():
            raise KeyError(f"no oracle record for {key}: regenerate tests/golden/oracle_records.json.gz")

    def _fold(self, *arrays):
        for a in arrays:
            self.h.update(np.ascontiguousarray(a).tobytes())
        self.n += 1
        if self.n % EVERY == 0:
            self._mark()

    def _mark(self):
        d = self.h.copy().hexdigest()[:16]
        i = len(self.marks)
        self.marks.append(d)
        if self.want is not None:
            assert i < len(self.want) and self.want[i] == d, \
                f"{self.key}: outputs differ from the oracle's between output {EVERY * i} and {self.n}"

    def observe(self):
        r, o, f = self.env.observe()
        self._fold(r, o["rgb"], f, *[self.env.info[k] for k in sorted(self.env.info)])
        return r, o, f

    def get_state(self, idx):
        b = self.env.get_state(idx)
        self._fold(np.frombuffer(b, np.uint8))
        return b

    def act(self, ac):
        self.env.act(ac)

    def set_state(self, idx, blob):
        self.env.set_state(idx, blob)

    def close(self):
        if self.env.h is None:
            return
        if self.n % EVERY:
            self._mark()
        self.env.close()
        if self.want is not None:
            assert len(self.want) == len(self.marks), f"{self.key}: {len(self.marks)} digests, the oracle recorded {len(self.want)}"
        else:
            with open(os.path.join(recording_dir(), re.sub(r"[^\w.-]", "_", self.key)[-150:] + ".json"), "w") as f:
                json.dump({self.key: self.marks}, f)

    def __getattr__(self, name):
        return getattr(self.env, name)


def oracle_env(num, env_name, lib_path, key=None, **kw):
    """The oracle on the stand-in pack while recording; else `lib_path` (the library under test) on it."""
    if recording_dir():
        kw.pop("extra_options", None)  # options of the library under test; the oracle takes its switches from the environment
        kw.pop("launch_shape", None)   # how the library under test cuts a step into launches: not an input of the outputs
        env = RefVecEnv(num, env_name, lib_path=REF_LIB, pack_path=STANDIN_PACK, **kw)
    else:
        env = RefVecEnv(num, env_name, lib_path=lib_path, resource_root=STANDIN_PACK, **kw)
    return Checked(env, _next_key(key))


def merge(record_dir, out=RECORDS, replace=False):
    """Add the records of a recording run (PG_ORACLE_RECORD_DIR) to `out`, keeping every record already in it.
    A key that is already there must come back with the same digests (re-recording an existing test is how
    a recording machine shows it reproduces the oracle); replace=True lets the new digests win instead.
    Returns (records in `out`, keys added, keys re-recorded identically)."""
    recs = {}
    if os.path.exists(out):
        with gzip.open(out, "rt") as f:
            recs = json.load(f)
    added, same, changed = [], [], []
    for fn in sorted(os.listdir(record_dir)):
        with open(os.path.join(record_dir, fn)) as f:
            for key, marks in json.load(f).items():
                if key not in recs:
                    added.append(key)
                elif recs[key] == marks:
                    same.append(key)
                else:
                    changed.append(key)
                    if not replace:
                        continue
                recs[key] = marks
    if changed and not replace:
        raise ValueError(f"{len(changed)} existing records would change (pass replace=True to overwrite): {changed[:8]}")
    with gzip.GzipFile(out, "wb", mtime=0) as f:
        f.write(json.dumps(recs, sort_keys=True, separators=(",", ":")).encode())
    return len(recs), added, same
