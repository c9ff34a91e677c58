"""Goldens of the tests that once ran the unmodified reference next to the product at test time (the reference reader,
AdjList on fuzz and tiled sets, AdjList on the reference's own unitig FASTA of config 1).  The reference binaries come
from `make -C oracle ref`; the inputs are the seeded sets the tests build, so the tests compare against these records
without the reference being present.  Writes ref_live.json (sha256 and length of every reference output) and
unitigs_cfg1_k<k>.fa.gz (the reference's unitigs that AdjList reads).

    python tests/golden/make_golden_ref_live.py
"""
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import overlap_cases as oc  # noqa: E402
import test_gpu_overlap as tgo  # noqa: E402
import test_host_overlap as tho  # noqa: E402
import test_host_reader as thr  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")


def digest(data: bytes) -> dict:
    return {"sha256": hashlib.sha256(data).hexdigest(), "bytes": len(data)}


def run(args, **kw):
    r = subprocess.run(args, capture_output=True, check=True, **kw)
    return r.stdout


def main():
    out = {}
    tmp = tempfile.mkdtemp(prefix="abyss_golden_live_")
    # the reference reader: records written by tests/test_host_reader.py
    paths = thr.write_reader_files(tmp)
    out["reader"] = digest(run([os.path.join(REF, "ref_arith"), "reads", "dump", *paths]))
    paths = thr.write_sam_qseq_files(tmp)
    out["reader_formats"] = {}
    for opts in thr.READER_OPTS:
        env = dict(os.environ, **{"REF_" + k: v for k, v in opts.items()})
        out["reader_formats"][thr.opts_key(opts)] = digest(run([os.path.join(REF, "ref_arith"), "reads", "dump", *paths], env=env))
    # AdjList on fuzz and tiled sets
    adj = os.path.join(REF, "AdjList-ref")
    out["adjlist"] = {}
    for c in tho.live_cases() + tgo.live_cases():
        fa = os.path.join(tmp, "in.fa")
        oc.write_fasta(c, fa)
        out["adjlist"][c["name"]] = digest(oc.normalise(run([adj] + oc.command_args(c, fa)), adj).replace(fa.encode(), b"IN.fa"))
    # AdjList on the reference's unitigs of config 1
    from abyss_b200.synth import ReadSet
    fq = os.path.join(tmp, "r.fq")
    ReadSet(1, 200000, 53333, 150, 0.005).write_fastq(fq)
    out["real_unitigs"] = {}
    for k, m, fmt in tho.REAL_UNITIG_SETS:
        gz = os.path.join(HERE, f"unitigs_cfg1_k{k}.fa.gz")
        if not os.path.exists(gz):
            fa = run(["bash", "-c", f"ulimit -s 65536; {os.path.join(REF, 'abyss-bloom-dbg-ref')} -k{k} --kc=2 -b64M -H4 -j1 {fq} 2>/dev/null"])
            with gzip.GzipFile(gz, "wb", mtime=0) as f:
                f.write(fa)
        fa = os.path.join(tmp, "unitigs-1.fa")
        with open(fa, "wb") as f:
            f.write(gzip.open(gz).read())
        got = run([adj, f"-k{k}", f"-m{m}", fmt, fa])
        out["real_unitigs"][f"k{k}_m{m}_{fmt[2:]}"] = digest(oc.normalise(got, adj).replace(fa.encode(), b"IN.fa"))
    # option aliases, several files, standard input
    out["adjlist_aliases"] = []
    for args, stdin in tho.alias_runs(tmp):
        got = run([adj] + args, input=stdin)
        out["adjlist_aliases"].append(digest(got.replace(tmp.encode(), b"TMP")))
    with open(os.path.join(HERE, "ref_live.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote ref_live.json")


if __name__ == "__main__":
    main()
