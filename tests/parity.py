"""The checks the reference-parity tests share: digests, the --read-log text, the assembler through the C ABI and through
abyss-bloom-dbg, the width tests' `abyss-bloom graph` and `trim` runs, and the host harnesses that run the kernels' templates
on one CPU thread.  Each check lives here once and asserts everything that any of its former copies asserted."""
import gzip
import hashlib
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "abyss_b200", "lib")
ORACLE = os.path.join("oracle", "abyss_oracle.c")
sys.path.insert(0, GOLD)
from make_golden_kwidth import blank_trace, raw_reads, reader_view, write_fastq  # noqa: E402


def _bytes(data):
    return data.encode() if isinstance(data, str) else data


def md5(data):
    return hashlib.md5(_bytes(data)).hexdigest()


def sha256(data):
    return hashlib.sha256(_bytes(data)).hexdigest()


def read_log(ids, codes):
    """the --read-log text of the assembler's read codes"""
    from abyss_b200.capi import READ_CODES
    return "read_id\tresult\n" + "".join(f"{i}\t{READ_CODES[c]}\n" for i, c in zip(ids, codes))


def counters_sha256(bloom_file):
    """sha256 of the counters of an `abyss-bloom build -t counting` file: the bytes after its header"""
    tag = b"[HeaderEnd]\n"
    return sha256(bloom_file[bloom_file.index(tag) + len(tag):])


def run(*cmd, cwd=None, env=None):
    """a command that must exit with status 0; its CompletedProcess (bytes)"""
    r = subprocess.run([str(c) for c in cmd], cwd=cwd, env=env, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return r


def check_unitigs(case, fasta, log, trace=None):
    """FASTA and read log (bytes or str) against the case's digests of the reference's; the -T trace too when given"""
    fasta = _bytes(fasta)
    assert fasta.count(b">") == case["n_contigs"]
    assert md5(fasta) == case["fasta_md5"]
    assert md5(log) == case["readlog_md5"]
    if trace is not None:
        assert sha256(blank_trace(trace)) == case["trace_sha256"]


# ---- the assembler through the C ABI ------------------------------------------------------------------------------------

def assemble(case, ids, seqs, batch=None):
    """the reads through a fresh counting filter and Assembler: (FASTA, read codes, abb_assembly_stats)"""
    from abyss_b200.capi import Assembler, Filter, pack_reads
    reads = seqs if isinstance(seqs, tuple) else pack_reads(seqs)
    f = Filter.counting(case["counters"], case["H"], case["k"], case["kc"], mask=case.get("mask", ""))
    f.insert_reads(reads)
    a = Assembler(f, read_log=True)
    fasta, codes = a.assemble(ids, reads, batch)
    st = a.stats()
    a.close()
    f.close()
    return fasta, codes, st


def check_assembler_c_abi(case, monkeypatch, reads=None, batch=997):
    """the counters, then the unitigs in one batch, in batches of `batch` reads and with ABB_NO_TILES=1; `reads` = (ids,
    sequences), by default the width cases' reads as the reference's reader sees them.  Returns the one-batch statistics."""
    from abyss_b200.capi import Filter
    ids, seqs = reads or map(list, zip(*reader_view(raw_reads(case["reads"]))))
    if "counters_sha256" in case:
        f = Filter.counting(case["counters"], case["H"], case["k"], case["kc"])
        f.insert_reads(seqs)
        assert sha256(f.download().tobytes()) == case["counters_sha256"]
        f.close()
    for b in (None, batch):
        fasta, codes, st = assemble(case, ids, seqs, b)
        check_unitigs(case, fasta, read_log(ids, codes))
        if b is None:
            one_batch = st
    monkeypatch.setenv("ABB_NO_TILES", "1")
    fasta, codes, _ = assemble(case, ids, seqs)
    check_unitigs(case, fasta, read_log(ids, codes))
    return one_batch


# ---- the command-line programs ------------------------------------------------------------------------------------------

def bloom_dbg_cli(case, reads, workdir, *opts, env=None):
    """abyss-bloom-dbg -k K --kc KC -b B -H H -j1 --read-log -T and `opts` on the file `reads`: (FASTA, read log, trace)"""
    fa, log, tr = (os.path.join(workdir, x) for x in ("out.fa", "read.log", "trace.tsv"))
    run(os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", *opts, f"--kc={case['kc']}", f"-b{case['b']}", f"-H{case['H']}", "-j1",
        f"--read-log={log}", "-T", tr, "-o", fa, reads, env=env)
    return open(fa, "rb").read(), open(log, "rb").read(), open(tr).read()


def check_counting_build(case, reads, workdir, env=None):
    """abyss-bloom build -t counting: the counters of the reference's file"""
    bf = os.path.join(workdir, "c.bloom")
    run(os.path.join(BIN, "abyss-bloom"), "build", "-k", case["k"], "-t", "counting", f"-b{case['counters']}", f"-H{case['H']}", bf, reads,
        env=env)
    assert counters_sha256(open(bf, "rb").read()) == case["counters_sha256"]


def check_assembler_cli(case, tmp_path, records=None, opts=None, env=None):
    """abyss-bloom-dbg on `records` (the width cases' reads by default) with the case's option or `opts`: FASTA, read log,
    trace and, where the case has them, the counters of `abyss-bloom build`"""
    fq = os.path.join(tmp_path, "reads.fq")
    write_fastq(raw_reads(case["reads"]) if records is None else records, fq)
    if opts is None:
        opts = [case["opt"]] if case.get("opt") else []
    check_unitigs(case, *bloom_dbg_cli(case, fq, tmp_path, *opts, env=env))
    if "counters_sha256" in case:
        check_counting_build(case, fq, tmp_path, env)


def check_dump(data, case, gz=None):
    """a dump or track against the case's size, line count and sha256, and against the reference's whole file where one is kept"""
    assert (len(data), data.count(b"\n")) == (case["bytes"], case["lines"])
    assert sha256(data) == case["sha256"]
    if gz and os.path.exists(gz):
        assert data == gzip.open(gz, "rb").read()


def check_dbg_graph(case, tmp_path, env=None):
    """abyss-bloom-dbg -g: the GraphViz dump of the width case's reads"""
    fq, dot = os.path.join(tmp_path, "reads.fq"), os.path.join(tmp_path, "g.dot")
    write_fastq(raw_reads(case["reads"]), fq)
    bloom_dbg_cli(case, fq, tmp_path, "-g", dot, "--batch-reads=700", env=env)
    check_dump(open(dot, "rb").read(), case)


def check_coverage_track(case, tmp_path, env=None):
    """abyss-bloom-dbg -C -R: the coverage track of the width case's reads over the genome they were drawn from"""
    from abyss_b200.synth import ReadSet
    from make_golden_covtrack import ref_fasta
    fq, ref, wig = (os.path.join(tmp_path, x) for x in ("reads.fq", "ref.fa", "cov.wig"))
    s = case["reads"]
    write_fastq(raw_reads(s), fq)
    ref_fasta(ReadSet.from_coverage(s["seed"], s["genome"], s["cov"], s["L"], s["err"]), ref)
    bloom_dbg_cli(case, fq, tmp_path, "-C", wig, "-R", ref, env=env)
    check_dump(open(wig, "rb").read(), case)


def abyss_bloom(*args, cwd=None, env=None):
    return subprocess.run([os.path.join(BIN, "abyss-bloom"), *map(str, args)], cwd=cwd, env=env, capture_output=True)


def build_filters(filters, cwd, env=None):
    """the `abyss-bloom` runs that write the filters a test directory needs"""
    for f in filters:
        r = abyss_bloom(*f["args"], cwd=cwd, env=env)
        assert r.returncode == 0, r.stderr.decode()


def check_bloom_graph_cli(case, cwd, gz, env=None):
    """`abyss-bloom graph`: exit status, stderr and the dump of the reference"""
    r = abyss_bloom(*case["args"], cwd=cwd, env=env)
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    check_dump(r.stdout, case, gz)


def check_trim_cli(case, cwd, env=None):
    """`abyss-bloom trim`: exit status, stderr and stdout of the reference"""
    r = abyss_bloom(*case["args"], cwd=cwd, env=env)
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert md5(r.stdout) == case["stdout_md5"]


# ---- host harnesses -----------------------------------------------------------------------------------------------------

def harness(name, *sources, flag=None):
    """a module-scoped fixture that compiles `sources` (paths from the repository's root) into the harness `name` once"""
    @pytest.fixture(scope="module")
    def exe(tmp_path_factory):
        out = str(tmp_path_factory.mktemp(name) / name)
        subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-pthread", *([flag] if flag else []), "-o", out,
                        *(os.path.join(ROOT, s) for s in sources)], check=True, capture_output=True)
        return out
    return exe


def run_host_walk(exe, case, reads, log=None, tiles=False, drop=None):
    """tests/host_walk on the case's k, kc, H, counters, trim (k by default) and mask, with tiles and with the tiles of
    seed `drop` dropped when asked: (FASTA, read log or None, stderr)"""
    env = {x: v for x, v in os.environ.items() if not x.startswith("HOST_WALK_")}
    env["HOST_WALK_MASK"] = case.get("mask", "")
    if tiles or drop is not None:
        env["HOST_WALK_TILES"] = "1"
    if drop is not None:
        env["HOST_WALK_DROP_TILES"] = str(drop)
    r = run(exe, case["k"], case["kc"], case["H"], case["counters"], case.get("trim", case["k"]), reads, *([log] if log else []), env=env)
    return r.stdout, open(log, "rb").read() if log else None, r.stderr.decode()


def check_host_assembler(exe, case, tmp_path, tiles):
    """the walk harness on a width case: the unitigs and read log of the reference"""
    fq, log = os.path.join(tmp_path, "reads.fq"), os.path.join(tmp_path, "read.log")
    write_fastq(reader_view(raw_reads(case["reads"])), fq)
    check_unitigs(case, *run_host_walk(exe, case, fq, log, tiles)[:2])


def check_host_bloom_graph(exe, case, cwd, gz):
    """tests/host_bloom_graph on the case's harness command line: the reference's dump"""
    check_dump(run(exe, *case["harness"], cwd=cwd).stdout, case, gz)


def check_host_trim(exe, case, cwd):
    """tests/host_trim on the case's harness command line: the reference's stdout and branch length threshold"""
    r = run(exe, *case["harness"], cwd=cwd)
    assert md5(r.stdout) == case["stdout_md5"]
    m = re.search(r"min length threshold for true branches \(k-mers\): (\d+)", case["stderr"])
    if m:
        assert f"minBranchLen {m.group(1)} " in r.stderr.decode()
