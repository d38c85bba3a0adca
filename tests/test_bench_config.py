"""CPU: both arms of bench.py print the identical `config` object for the same flags."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_config_dict_is_shared_by_both_arms():
    import inspect
    import bench
    src = inspect.getsource(bench)
    # every JSON line builds its config through make_config with the same in-flight default
    assert src.count('"config": make_config(') >= 3
    a = bench.make_config("0075", True)
    b = bench.make_config("0075", True, 4)
    assert a == b and a["frames_in_flight_per_gpu"] == 4 and "0.075 m" in a["workload"]
    assert bench.make_config("01", True)["workload"] != a["workload"]
