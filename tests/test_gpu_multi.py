"""Multi-GPU tests of the exact position-sharded pass 1 (they need 2 or more GPUs and skip with one).
At every world size the counters must be the sequential -j1 array bit for bit (sha256 of the reference's
`abyss-bloom build -t counting` output, tests/golden/e2e_cases.json) and the unitig FASTA byte-identical to the
reference's (tests/golden/*.fa) -- the same goldens the single-GPU tests use."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys, json, hashlib, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
from abyss_b200 import capi
from abyss_b200.synth import ReadSet
os.environ["ABB_SHARD_MIN_WORLD"] = "2"  # the position-sharded insert also at world size 2 (the library default keeps 2 ranks replicated)
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
dev = torch.device("cuda", rank)
def bcast(b):
    box = [b]; dist.broadcast_object_list(box, src=0); return box[0]
comm = capi.Comm(rank, world, rank, bcast)
gd = os.path.join(%(root)r, "tests", "golden")
cases = {c["name"]: c for c in json.load(open(os.path.join(gd, "e2e_cases.json")))}
for name, window in (("e2e_g20k_k32", 0), ("e2e_g30k_k64", 4096), ("e2e_g10k_k25_small", 1000)):
    c = cases[name]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    L = c["L"]
    asc = rs.ascii(0, rs.n)
    bases = torch.from_numpy(asc.reshape(-1).copy()).to(dev)
    offs = torch.arange(rs.n + 1, dtype=torch.int64, device=dev) * L
    f = capi.Filter.counting(c["counters"], c["H"], c["k"], c["kc"], device=rank)
    if window:
        f.set_window(window)
    nk = f.insert_reads_sharded_dev(comm, bases.data_ptr(), offs.data_ptr(), rs.n)
    assert nk == rs.n * (L - c["k"] + 1), (nk, rs.n)
    got = f.download()
    assert hashlib.sha256(got.tobytes()).hexdigest() == c["counters_sha256"], f"{name}: rank {rank} counters differ from the -j1 reference"
    # host-buffer entry point gives the same
    g = capi.Filter.counting(c["counters"], c["H"], c["k"], c["kc"], device=rank)
    g.insert_reads_sharded(comm, capi.fixed_length_reads(asc))
    assert (g.download() == got).all()
    g.close()
    # pass 2 with classification, candidate scans and tile production sharded over the ranks: FASTA and read log
    # identical to the reference on every rank
    a = capi.Assembler(f, read_log=True)
    a.set_comm(comm)
    out = a.process_reads_dev(bases.data_ptr(), offs.data_ptr(), rs.n)
    fasta = "".join(f">{i} {len(s)} {cov} read:{rs.read_id(r)}\n{s}\n" for i, (r, s, cov) in enumerate(out))
    assert fasta == open(os.path.join(gd, name + ".fa")).read(), f"{name}: rank {rank} FASTA differs"
    res = a.read_results()
    log = open(os.path.join(gd, name + ".readlog.tsv")).read().split("\n")[1:-1]
    assert [f"{rs.read_id(i)}\t{capi.READ_CODES[res[i]]}" for i in range(rs.n)] == log
    a.close(); f.close()
dist.barrier()
if rank == 0:
    print("MULTI_OK")
dist.destroy_process_group()
'''


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_insert_is_exact(tmp_path, world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    w = tmp_path / "worker.py"
    w.write_text(WORKER % {"root": ROOT})
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(29541 + world), str(w)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "MULTI_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.parametrize("ndev", [2, 8])
def test_cli_devices_option(tmp_path, ndev):
    # abyss-bloom-dbg --devices=0-(N-1): the C++ host drives N GPUs (one thread per GPU, NCCL behind the C ABI) and
    # prints the same bytes as the reference / the single-GPU run
    import json
    import torch
    from abyss_b200 import build
    from abyss_b200.synth import ReadSet
    if torch.cuda.device_count() < ndev:
        pytest.skip(f"needs {ndev} GPUs")
    build.build()
    gd = os.path.join(ROOT, "tests", "golden")
    c = {x["name"]: x for x in json.load(open(os.path.join(gd, "e2e_cases.json")))}["e2e_g20k_k32"]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    fq = str(tmp_path / "r.fq")
    rs.write_fastq(fq)
    fa, log = str(tmp_path / "out.fa"), str(tmp_path / "read.log")
    for policy in ({"ABB_SHARD_MIN_WORLD": "2"}, {}):  # sharded insert forced / the library's own choice for this world size
        r = subprocess.run([os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom-dbg"), f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}",
                            f"--devices=0-{ndev - 1}", "--batch-reads=1500", f"--read-log={log}", "-o", fa, fq], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, **policy))
        assert r.returncode == 0, r.stderr
        assert open(fa).read() == open(os.path.join(gd, "e2e_g20k_k32.fa")).read()
        assert open(log).read() == open(os.path.join(gd, "e2e_g20k_k32.readlog.tsv")).read()
