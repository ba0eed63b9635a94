"""bench.py pieces that run without a GPU: the clock sampler degrades to an explicit "no sampler" record instead of failing,
--dump-outputs writes the solution as float64 arrays within its size budget."""
import importlib.util
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_bench():
    spec = importlib.util.spec_from_file_location("bench_module", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_clock_sampler_without_nvml_or_nvidia_smi():
    bench = load_bench()
    sampler = bench.ClockSampler(0)
    sampler.start()
    mark = sampler.mark()
    rec = sampler.stop(mark, sampler.mark())
    assert set(rec) >= {"sm_mhz", "sm_max_mhz", "reasons", "samples"}
    assert rec["samples"] == 0 or rec["sm_mhz"] is not None  # either nothing could be sampled (this box) or real samples


def test_dump_outputs_writes_the_solution_as_float64(tmp_path):
    import numpy as np

    from whatshap_b200._abi import FlatSolution

    bench = load_bench()
    sol = FlatSolution(5, 3, 1)
    sol.cost = 4294967295
    sol.path_index[:] = [0, 1, 2, 3, 4]
    sol.partition[:] = [1, 0, 1]
    bench.dump_outputs(str(tmp_path), sol)
    got = {p.stem: np.load(p) for p in tmp_path.glob("*.npy")}
    assert set(got) == {"cost", "path_index", "path_tv", "partition", "sr_allele", "sr_quality"}
    assert all(a.dtype == np.float64 for a in got.values())
    assert got["cost"].tolist() == [4294967295.0] and got["path_index"].tolist() == [0, 1, 2, 3, 4]
    assert got["sr_allele"].shape == (1, 2, 5)
    bench.DUMP_BUDGET = 6 * 16  # two float64 values per array: larger arrays become a fixed sample of their elements
    bench.dump_outputs(str(tmp_path), sol)
    a, b = np.load(tmp_path / "path_index.npy"), np.load(tmp_path / "sr_allele.npy")
    assert a.shape == (2,) and set(a.tolist()) <= {0, 1, 2, 3, 4} and b.shape == (2,)
    bench.dump_outputs(str(tmp_path), sol)
    assert np.array_equal(np.load(tmp_path / "path_index.npy"), a)
