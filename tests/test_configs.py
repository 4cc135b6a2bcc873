"""The encoder configurations the benchmark and the tests run, pinned to the reference's configuration files (config_*.txt in the reference's
root: `-key value ; comment` lines).  bench.CONFIGS names, for each BASELINE.json configuration, the file its flags stand for; the flags must be
exactly that file's options, so the benchmark and the RD-loop tests that import them run what the configuration says.  CPU only; skipped where
the reference's sources are absent (the default place is oracle/Makefile's REF)."""
import os

import pytest

import bench
import test_dropin_link

REF_SRC = os.environ.get("THOR_REFERENCE", "/root/reference")

needs_src = pytest.mark.skipif(not os.path.exists(os.path.join(REF_SRC, "config_HDB_high_efficiency.txt")),
                               reason="the reference's configuration files are not on this machine")


def options_of_file(name):
    """{key: value} of a reference configuration file; a key given twice is an error"""
    out = {}
    for line in open(os.path.join(REF_SRC, name + ".txt")):
        line = line.split(";", 1)[0].split()
        if not line:
            continue
        assert len(line) == 2 and line[0].startswith("-"), (name, line)
        assert line[0] not in out, (name, "option given twice", line[0])
        out[line[0]] = line[1]
    return out


def options_of_flags(flags):
    """{key: value} of a Thorenc command line; a key given twice is an error"""
    flags = flags.split() if isinstance(flags, str) else list(flags)
    assert len(flags) % 2 == 0, flags
    keys = flags[0::2]
    assert all(k.startswith("-") for k in keys) and len(set(keys)) == len(keys), flags
    return dict(zip(keys, flags[1::2]))


@needs_src
@pytest.mark.parametrize("config", sorted(bench.CONFIGS))
def test_bench_config_flags_are_the_reference_file(config):
    flags, cfgfile = bench.CONFIGS[config][4], bench.CONFIGS[config][5]
    assert options_of_flags(flags) == options_of_file(cfgfile)


@needs_src
@pytest.mark.parametrize("name,cfgfile", [("HDB", "config_HDB_high_efficiency"), ("LDB", "config_LDB_low_complexity")])
def test_test_flags_are_the_reference_file(name, cfgfile):
    assert options_of_flags(getattr(test_dropin_link, name)) == options_of_file(cfgfile)


def test_test_flags_are_the_bench_flags():
    """without the reference's files: the tests' HDB and LDB are the benchmark's"""
    assert options_of_flags(test_dropin_link.HDB) == options_of_flags(bench.HDB)
    assert options_of_flags(test_dropin_link.LDB) == options_of_flags(bench.LDB)
