"""Regenerate the committed golden outputs from the compiled reference (oracle/Makefile builds it where its sources are).

    python tests/golden/make_golden.py            # golden PAFs / GFF / ... and the stored reference answers
    python tests/golden/make_golden.py --answers  # the stored reference answers only

Writes tests/golden/DPP3_default.paf (+ option variants) and synthetic 'tiny'/'tiny5' PAFs: the reference ships no
expected outputs (SURVEY.md section 4), so these files ARE the golden vectors; md5 of the default DPP3 PAF is
74fd00200bda6c03380bb3062fb5178b (SURVEY.md App. D).

Then tests/golden/reference_calls.json.gz, every answer of the reference the tests compare with (tests/oracle_lib.py
reference()): the CPU tests that ask it are run once against oracle/_ref/libref.so, and the reference CLI is run on the inputs
of the GPU parity tests (test_gpu_e2e, test_gpu_dropin, test_gpu_index_options, test_gpu_configs; a few minutes for the 1 Gbp
C3s shape).
"""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from miniprot_b200 import synth  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "miniprot")
RECORDED_TESTS = ["tests/test_oracle_pin.py", "tests/test_emu_nasw.py", "tests/test_tables.py",
                  # the reference's tables and DP answers under every -T, and its -T<n> -d index files (test_gpu_trans_code too)
                  "tests/test_host_trans_code.py::test_emu_trans_code", "tests/test_host_trans_code.py::test_host_index_trans_code"]


def run(args, out):
    with open(out, "wb") as f:
        subprocess.run([REF, "-t4"] + args, check=True, stdout=f, stderr=subprocess.DEVNULL)


def goldens(d):
    g, p = os.path.join(HERE, "DPP3-hs.gen.fa.gz"), os.path.join(HERE, "DPP3-mm.pep.fa.gz")
    run([g, p], os.path.join(HERE, "DPP3_default.paf"))
    run(["-j2", g, p], os.path.join(HERE, "DPP3_j2.paf"))
    run(["-G", "2k", g, p], os.path.join(HERE, "DPP3_G2k.paf"))
    for cfg in ("tiny", "tiny5"):
        gg, pp = synth.generate(synth.CONFIGS[cfg], d)
        run([gg, pp], os.path.join(HERE, cfg + ".paf"))
    # the other output formats (format.c:189-452), on the set that exercises every CIGAR operation, and on DPP3
    gg, pp = synth.generate(synth.CONFIGS["tiny5"], d)
    for name, args in (("gff", ["--gff"]), ("gtf", ["--gtf"]), ("aln", ["--aln"]), ("trans", ["--trans", "-u"]), ("gff_only", ["--gff-only", "--gff-delim", "#"])):
        run(args + [gg, pp], os.path.join(HERE, "tiny5_" + name + ".txt"))
        run(args + [g, p], os.path.join(HERE, "DPP3_" + name + ".txt"))


def answers(d):
    env = dict(os.environ, MPB_RECORD_REFERENCE="1")
    rec = os.path.join(HERE, "reference_calls.json.gz")
    if os.path.exists(rec):
        os.remove(rec)
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", *RECORDED_TESTS], cwd=ROOT, env=env, check=True)
    os.environ["MPB_RECORD_REFERENCE"] = "1"
    import oracle_lib as ol
    import test_gpu_configs
    import test_gpu_e2e

    ol.RECORDING = True
    ol._answers()
    for cfg, args, _ in test_gpu_e2e.SMALL_CASES:
        g, p = synth.generate(synth.CONFIGS[cfg], os.path.join(d, cfg))
        ol.ref_cli(list(args), g, p, os.cpu_count() or 8)
    import test_gpu_dropin

    ol.ref_index_file(synth.generate(synth.CONFIGS["tiny"], os.path.join(d, "tiny"))[0])
    for g in (test_gpu_dropin.write_odd_fasta(os.path.join(d, "odd.fa")), ol.DPP3_GENOME, synth.generate(synth.CONFIGS["small"], os.path.join(d, "small"))[0]):
        ol.ref_index_file(g)
    import test_gpu_index_options

    for g in (test_gpu_dropin.write_odd_fasta(os.path.join(d, "odd.fa")), synth.generate(synth.CONFIGS["tiny"], os.path.join(d, "tiny"))[0]):
        for opts in test_gpu_index_options.INDEX_SETS:
            ol.ref_index_file(g, opts)
    for g, p in test_gpu_dropin.map_inputs(os.path.join(d, "tiny")):
        test_gpu_dropin.ref_regions(g, p)
    for g, p, _, args, _ in test_gpu_dropin.spsc_inputs(d):
        ol.ref_cli(list(args), g, p, os.cpu_count() or 8)
    for cfg, opts in test_gpu_configs.CASES.items():
        g, p = synth.generate(synth.CONFIGS[cfg], os.path.join(d, cfg))
        for o in opts:
            print(cfg, repr(o), ol.ref_cli(o.split(), g, p, os.cpu_count() or 8), flush=True)


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as d:
        if "--answers" not in sys.argv:
            goldens(d)
        answers(d)
