"""The measured tuning table: parsing, range lookup, fall-through (host only)."""
import gloo_b200 as gb

cu = gb._C.cuda

TABLE = """
# comment line
allreduce P=8 buf=sym maxbytes=16384 algo=ll blocks=4
allreduce P=8 buf=sym maxbytes=262144 algo=one_shot blocks=8   # trailing comment
allreduce P=8 buf=sym maxbytes=inf algo=nvls blocks=148 unroll=8
allreduce P=8 buf=user maxbytes=inf algo=pipelined blocks=128 tile=1024
allgather P=8 buf=reg maxbytes=4096 algo=ll blocks=0
allgather P=8 buf=reg maxbytes=inf algo=push blocks=222
this line is garbage
allreduce P=x buf=sym maxbytes=1 algo=ll blocks=1
"""


def test_parse_lookup_and_dump():
    cu.tuning_clear()
    try:
        assert cu.tuning_load_string(TABLE) == 6
        e = cu.tuning_lookup("allreduce", 8, 0, 1000)
        assert e["algo"] == "ll" and e["blocks"] == 4
        assert cu.tuning_lookup("allreduce", 8, 0, 16384)["algo"] == "ll"
        assert cu.tuning_lookup("allreduce", 8, 0, 16385)["algo"] == "one_shot"
        big = cu.tuning_lookup("allreduce", 8, 0, 400_000_000)
        assert big["algo"] == "nvls" and big["blocks"] == 148 and big["unroll"] == 8
        assert cu.tuning_lookup("allreduce", 8, 2, 1 << 20)["tile"] == 1024
        assert cu.tuning_lookup("allreduce", 4, 0, 1000) is None      # no group for P=4
        assert cu.tuning_lookup("allreduce", 8, 1, 1000) is None      # no group for registered buffers
        assert cu.tuning_lookup("allgather", 8, 1, 100)["algo"] == "ll"
        dump = cu.tuning_dump()
        assert "allreduce P=8 buf=sym maxbytes=inf algo=nvls blocks=148 unroll=8" in dump
        cu.tuning_clear()
        assert cu.tuning_load_string(dump) == 6  # round trip
    finally:
        cu.tuning_clear()


def test_packaged_table_parses():
    import os

    path = os.path.join(os.path.dirname(gb.__file__), "tuning", "h100.tune")
    if not os.path.exists(path):
        return
    cu.tuning_clear()
    try:
        assert cu.tuning_load_file(path) > 0
    finally:
        cu.tuning_clear()


def test_packaged_table_is_complete_and_sane():
    """Every line of the packaged table parses (no silently dropped rows), every (collective, P, kind) group is
    sorted and ends with maxbytes=inf, and the algorithm names are ones the selector knows."""
    import os

    path = os.path.join(os.path.dirname(gb.__file__), "tuning", "h100.tune")
    lines = [ln.split("#")[0].strip() for ln in open(path)]
    lines = [ln for ln in lines if ln]
    cu.tuning_clear()
    try:
        assert cu.tuning_load_file(path) == len(lines)
    finally:
        cu.tuning_clear()
    known = {"allreduce": {"ll", "one_shot", "two_shot", "nvls", "hybrid", "pipelined"},
             "broadcast": {"push", "relay", "nvls", "scatter", "direct"}}
    groups = {}
    for ln in lines:
        f = ln.split()
        kv = dict(x.split("=", 1) for x in f[1:])
        groups.setdefault((f[0], kv["P"], kv["buf"]), []).append(kv)
        if f[0] in known:
            assert kv["algo"] in known[f[0]], ln
    for key, rows in groups.items():
        bounds = [float("inf") if r["maxbytes"] == "inf" else float(r["maxbytes"]) for r in rows]
        assert bounds == sorted(bounds) and bounds[-1] == float("inf"), key
        assert len(set(bounds)) == len(bounds), key


def test_merge_tables_splices_from_min_bytes_up():
    from gloo_b200.tune import merge_tables

    base = ["# header", "allreduce P=8 buf=sym maxbytes=4096 algo=ll blocks=1",
            "allreduce P=8 buf=sym maxbytes=inf algo=nvls blocks=32 unroll=2",
            "allreduce P=8 buf=reg maxbytes=inf algo=two_shot blocks=148 unroll=2",
            "broadcast P=8 buf=reg maxbytes=inf algo=push blocks=64"]
    new = ["# focus run", "allreduce P=8 buf=sym maxbytes=50000000 algo=nvls blocks=8 unroll=4",
           "allreduce P=8 buf=sym maxbytes=inf algo=nvls blocks=16 unroll=4",
           "allreduce P=4 buf=sym maxbytes=inf algo=hybrid blocks=64 unroll=32 tile=500"]
    out = merge_tables(base, new, 1 << 20)
    assert out[0] == "# header" and out[1] == base[1]
    assert out[2] == "allreduce P=8 buf=sym maxbytes=1048575 algo=nvls blocks=32 unroll=2"   # the straddling row keeps its lower part
    assert out[3:5] == new[1:3]
    assert base[3] in out and base[4] in out                                                  # other groups untouched
    assert out[-1] == new[3]                                                                  # a group the base did not have
    cu.tuning_clear()
    try:
        assert cu.tuning_load_string("\n".join(out)) == 7
        assert cu.tuning_lookup("allreduce", 8, 0, 400_000_000)["blocks"] == 16
        assert cu.tuning_lookup("allreduce", 8, 0, 2_000_000)["blocks"] == 8
        assert cu.tuning_lookup("allreduce", 8, 0, 500_000)["blocks"] == 32
    finally:
        cu.tuning_clear()
