"""CPU test of the keyed jobs on several devices (gpu.devices): NaiveTrain, ItemModelTrain and ItemModelTest cut their keys into one
contiguous range per device and run the single-device library call of each range on its own thread.  The jobs are linked against the
test doubles of the device library (tests/fake_device/*.c), whose numbers are per-key hashes of the key's own rows, independent of
where the rows sit in the arrays: so every output tree must be byte-identical for gpu.devices = 0, 0,1 and 0,1,2 (and for more
devices than keys).  The shard helper's balance is checked directly.  Set MLEASE_TEST_SANITIZE=thread to build under TSan."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
HOST = os.path.join(ROOT, "ml-ease_b200", "host")
FAKE = os.path.join(ROOT, "tests", "fake_device")


def _san():
    san = os.environ.get("MLEASE_TEST_SANITIZE", "")
    return ["-g", "-fsanitize=" + san, "-fno-omit-frame-pointer"] if san else []


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    import ctypes as C
    d = tmp_path_factory.mktemp("fakehost_shards")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared"] + _san() + ["-o", so] +
                          [os.path.join(HOST, f) for f in ("avro_io.cpp", "regression_jobs.cpp", "item_model_jobs.cpp", "item_model_train_job.cpp")] +
                          ["-x", "c"] + [os.path.join(FAKE, f) for f in ("fake_mlease_b200.c", "fake_item_model.c", "fake_item_model_train.c")] +
                          ["-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _cfg(path, kv):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
    return str(path)


def _run(h, job, cfg):
    assert h.mlease_job_run(job.encode(), cfg.encode()) == 0, h.mlease_job_last_error().decode()


def _bytes(root):
    """relative path -> raw bytes of every avro file under root, its random 16-byte sync marker (which also ends the file) zeroed."""
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith(".avro"):
                p = os.path.join(dp, f)
                data = open(p, "rb").read()
                out[os.path.relpath(p, root)] = data.replace(data[-16:], bytes(16))
    return out


def _models(path, keys, names):
    schema = {"type": "record", "name": "LinearModelAvro", "fields": [{"name": "key", "type": "string"}, {"name": "model", "type": {"type": "array", "items": {
        "type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"}, {"name": "value", "type": "float"}]}}}]}
    au.write_avro(path, schema, [{"key": k, "model": [{"name": "(INTERCEPT)", "term": "", "value": 0.25}] +
                                  [{"name": nm, "term": "", "value": 0.1 * (i + 1)} for i, nm in enumerate(names)]} for k in keys])


DEVICE_LISTS = ("0", "0,1", "0,1,2", ",".join(str(i) for i in range(40)))   # the last: more devices than keys


def test_keyed_job_trees_do_not_depend_on_the_device_count(fake_host, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(n) for n in npz["feature_names"]]
    # 13 keys of very different sizes (key 12 has 1 row), so that the cuts fall between unequal keys
    recs = au.fixture_records(npz, with_key=lambda i: min(12, int(np.sqrt(i) // 2.5)))
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, block=200)
    _run(fake_host, "RegressionPrepare", _cfg(tmp_path / "p.job", {"input.paths": tmp_path / "in", "output.path": tmp_path / "prep", "map.key": "pkey",
                                                                   "num.blocks": 2}))
    _models(str(tmp_path / "models" / "part-r-00000.avro"), ["1.0#%d" % k for k in range(0, 13, 2)] + ["10.0#%d" % k for k in range(1, 13, 3)], names[:20])
    trees = {}
    for devs in DEVICE_LISTS:
        tag = "d" + str(devs.count(",") + 1)
        base = tmp_path / tag
        _run(fake_host, "NaiveTrain", _cfg(tmp_path / (tag + "_n.job"), {"input.paths": tmp_path / "prep", "output.base.path": base / "naive", "num.blocks": 13,
                                                                         "lambda": "10,1", "data.size.threshold": 3, "remove.tmp.dir": "false",
                                                                         "gpu.devices": devs}))
        _run(fake_host, "ItemModelTrain", _cfg(tmp_path / (tag + "_i.job"), {"input.paths": tmp_path / "prep", "output.model.path": base / "imt",
                                                                             "intercept.lambdas": "1e-4,1", "default.lambdas": "0.1,2", "compute.var": "true",
                                                                             "intercept.default.prior.mean": 0.3, "gpu.devices": devs}))
        _run(fake_host, "ItemModelTest", _cfg(tmp_path / (tag + "_t.job"), {"input.paths": tmp_path / "in", "output.base.path": base / "imtest",
                                                                            "model.path": tmp_path / "models", "item.key": "pkey", "lambda": "1,10.0",
                                                                            "gpu.devices": devs}))
        trees[devs] = _bytes(base)
    one = trees["0"]
    assert sorted(one) == ["imt/models/part-r-00000.avro", "imtest/lambda-1/part-r-00000.avro", "imtest/lambda-10.0/part-r-00000.avro",
                           "naive/final-model/part-r-00000.avro", "naive/models/part-r-00000.avro"], sorted(one)
    for devs, t in trees.items():
        assert sorted(t) == sorted(one), devs
        for k in one:
            assert t[k] == one[k], (devs, k)


def test_item_model_test_shards_whose_keys_own_no_rows(fake_host, tmp_path):
    """ItemModelTest with 2 and 8 devices when one key holds 990 of the 1000 rows: the cost balance puts that key in a shard of its
    own and leaves shards with no key.  (A failing shard is tested on the GPU: these test doubles never fail.)"""
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(n) for n in npz["feature_names"]]
    recs = au.fixture_records(npz, with_key=lambda i: 0 if i < 990 else i - 989)[:1000]
    au.write_avro(str(tmp_path / "in" / "p.avro"), au.pig_schema_with_key(), recs)
    _models(str(tmp_path / "models" / "m.avro"), ["1.0#0", "1.0#3"], names[:5])
    trees = {}
    for devs in ("0", "0,1", "0,1,2,3,4,5,6,7"):
        out = tmp_path / ("o" + str(devs.count(",")))
        _run(fake_host, "ItemModelTest", _cfg(tmp_path / "t.job", {"input.paths": tmp_path / "in", "output.base.path": out, "model.path": tmp_path / "models",
                                                                   "item.key": "pkey", "lambda": "1", "gpu.devices": devs}))
        trees[devs] = _bytes(out)
    assert trees["0"] == trees["0,1"] == trees["0,1,2,3,4,5,6,7"]


@pytest.fixture(scope="module")
def shard_tool(tmp_path_factory):
    d = tmp_path_factory.mktemp("shardtool")
    src = d / "shard.cpp"
    src.write_text(r'''
#include <cstdio>
#include "jobs_common.hpp"
int main() {
  int K, D, n;
  if (scanf("%d %d %d", &K, &D, &n) != 3) return 2;
  std::vector<int64_t> krs(K + 1), rp;
  for (auto& x : krs) if (scanf("%ld", &x) != 1) return 2;
  rp.resize(krs[K] + 1);
  for (auto& x : rp) if (scanf("%ld", &x) != 1) return 2;
  for (int c : mlease_jobs::shard_keys(krs, rp, D, n)) printf("%d ", c);
  printf("\n");
  return 0;
}
''')
    exe = str(d / "shard")
    subprocess.check_call(["g++", "-O1", "-std=c++17"] + _san() + ["-I", HOST, "-o", exe, str(src), "-pthread"])
    return exe


@pytest.mark.parametrize("seed,K,nshards", [(0, 50, 3), (1, 7, 7), (2, 5, 9), (3, 400, 8), (4, 1, 2)])
def test_shard_keys_cuts_contiguous_balanced_ranges(shard_tool, seed, K, nshards):
    rng = np.random.default_rng(seed)
    D = 30
    rows = rng.integers(0, 40, K) * (rng.random(K) < 0.8)          # some keys have no rows
    rows[rng.integers(0, K)] = 300                                   # one heavy key
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    nnz = rng.integers(0, 12, krs[-1])
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    inp = "%d %d %d\n%s\n%s\n" % (K, D, nshards, " ".join(map(str, krs)), " ".join(map(str, rp)))
    cuts = [int(x) for x in subprocess.check_output([shard_tool], input=inp.encode()).split()]
    assert len(cuts) == nshards + 1 and cuts[0] == 0 and cuts[-1] == K
    assert all(a <= b for a, b in zip(cuts, cuts[1:]))               # contiguous, covering every key once
    cost = rows * float(D + 1) ** 2 + (rp[krs[1:]] - rp[krs[:-1]])
    shard = [cost[a:b].sum() for a, b in zip(cuts, cuts[1:])]
    assert max(shard) <= cost.sum() / nshards + cost.max() + 1e-6, (shard, cost.max())
