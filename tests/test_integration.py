"""The drop-in, exercised: the UNMODIFIED reference built against libhtsgpu.so
(integration/build_hts_gpu.sh: bgzf.c with integration/htsgpu_bgzf.patch and -DHAVE_HTSGPU, the
htscodecs entropy coders resolved to libhtsgpu.so) runs the reference's own test programs —
test/test_bgzf.c, test/test_view.c, bgzip — and must behave exactly like the stock build
(oracle/_ref) on the reference's fixtures.  SURVEY.md §8 rows a3 / a4 / a7 / (b); BASELINE config 1."""
import hashlib
import os
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = os.path.join(ROOT, "oracle", "_ref", "integration")
G = os.path.join(ROOT, "tests", "golden", "htslib")
have = os.path.exists(os.path.join(B, "test_view")) and os.path.exists(os.path.join(B, "stock", "test_view"))


def run(cmd, **kw):
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=600, **kw)


def test_patch_is_a_patch_not_a_copy():
    """integration/ holds a diff against the reference's bgzf.c, not the file"""
    p = open(os.path.join(ROOT, "integration", "htsgpu_bgzf.patch")).read()
    assert p.startswith("--- ") and "HAVE_HTSGPU" in p
    added = [l for l in p.splitlines() if l.startswith("+") and not l.startswith("+++")]
    context = [l for l in p.splitlines() if l.startswith(" ")]
    assert len(added) > 150 and len(context) < 120


@pytest.mark.skipif(not os.path.isdir("/root/reference"), reason="needs the reference tree to rebuild")
def test_integration_build_links_the_gpu_symbols():
    r = run(["bash", os.path.join(ROOT, "integration", "build_hts_gpu.sh")])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    out = r.stdout.decode()
    for sym in ("hgpu_bgzf_inflate_jobs_host", "rans_uncompress_4x16", "tok3_decode_names", "fqz_decompress", "arith_uncompress_to"):
        assert "from libhtsgpu.so: " + sym in out, out
    # the stock entropy coders are not in the GPU build
    nm = run(["nm", "-D", "--defined-only", os.path.join(B, "libhts_gpu.so")]).stdout.decode()
    assert " rans_uncompress_to_4x16" not in nm and " bgzf_mt" in nm


gpu = pytest.mark.gpu
need = pytest.mark.skipif(not have, reason="oracle/_ref/integration not built (needs the reference sources)")


@gpu
@need
def test_reference_test_bgzf_passes_on_the_gpu_build():
    r = run([os.path.join(B, "test_bgzf"), os.path.join(G, "bgziptest.txt")], cwd=B)
    assert r.returncode == 0, (r.stdout + r.stderr).decode()[-3000:]


@gpu
@need
@pytest.mark.parametrize("threads", [0, 4])
def test_bgzip_decompress_baseline_config1(threads):
    """BASELINE.json configs[0]: bgzip -d of test/bgziptest.txt.gz"""
    cmd = [os.path.join(B, "bgzip"), "-dc"] + (["-@", str(threads)] if threads else []) + [os.path.join(G, "bgziptest.txt.gz")]
    r = run(cmd)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == open(os.path.join(G, "bgziptest.txt"), "rb").read()


def _view(exe, args):
    r = run([exe] + args)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r.stdout


FILES = [("range.bam", []), ("colons.bam", []), ("bgzf_boundaries/bgzf_boundaries1.bam", []), ("bgzf_boundaries/bgzf_boundaries2.bam", []),
         ("bgzf_boundaries/bgzf_boundaries3.bam", []),
         ("ce#1000.v31.cram", ["-i", "reference=ce.fa"]), ("ce#1000.v30.cram", ["-i", "reference=ce.fa"]), ("ce#1000.v31arith.cram", ["-i", "reference=ce.fa"]),
         ("ce#1000.v31fqz.cram", ["-i", "reference=ce.fa"]), ("ce#5b_java.cram", ["-i", "reference=ce.fa"]), ("range.cram", ["-i", "reference=ce.fa"])]


@gpu
@need
@pytest.mark.parametrize("threads", [0, 4])
@pytest.mark.parametrize("name,extra", FILES)
def test_test_view_matches_the_stock_build(name, extra, threads):
    """test_view (sam_read1 -> SAM text) on the GPU build == the stock build, byte for byte"""
    path = os.path.join(G, name)
    if not os.path.exists(path):
        pytest.skip("fixture not imported")
    args = (["-@", str(threads)] if threads else [])
    for e in extra:                                 # the reference's own harness passes -i reference=<fa> (test/test.pl:823)
        args.append("reference=" + os.path.join(G, e[len("reference="):]) if e.startswith("reference=") else e)
    want = _view(os.path.join(B, "stock", "test_view"), args + [path])
    got = _view(os.path.join(B, "test_view"), args + [path])
    assert hashlib.md5(got).hexdigest() == hashlib.md5(want).hexdigest()
    assert len(got) > 100


@gpu
@need
def test_view_large_bam_through_the_batched_reader(tmp_path):
    """a BAM large enough for several HTSGPU_BATCH flushes (and a seek-free sequential read with 4 threads)"""
    import sys
    sys.path.insert(0, ROOT)
    from tools import synth
    corpus = synth.bam_bgzf_corpus(60e6, procs=4)
    hdr_txt = b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:248956422\n"
    import struct
    hdr = b"BAM\1" + struct.pack("<i", len(hdr_txt)) + hdr_txt + struct.pack("<i", 1) + struct.pack("<i", 5) + b"chr1\0" + struct.pack("<i", 248956422)
    p = tmp_path / "big.bam"
    with open(p, "wb") as f:
        f.write(synth.bgzf_block(hdr))
        f.write(corpus["comp"].tobytes())
        f.write(synth.BGZF_EOF)
    want = _view(os.path.join(B, "stock", "test_view"), ["-@", "4", str(p)])
    got = _view(os.path.join(B, "test_view"), ["-@", "4", str(p)])
    assert hashlib.md5(got).hexdigest() == hashlib.md5(want).hexdigest()
    assert got.count(b"\n") > 150000
