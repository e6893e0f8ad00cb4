#!/usr/bin/env python
"""Generates the fixtures under tests/golden/ from a speedseq checkout (its path in
SPEEDSEQ_CHECKOUT); the tests only read the committed outputs.

  ex_ref.fa.gz            the reference's example FASTA (example/data/human_g1k_v37_20_42220611-42542245.fasta), gzip'd
  ex_index.sha256.json    sha256 + size of the reference's own golden index files for that FASTA
                          (example/data/*.fasta.{amb,ann,pac,bwt,sa}) — the ONLY reference-owned known-answer data for
                          this path (SURVEY.md §8c); the oracle's and the product's index builders must reproduce them.
  ex_reads_2k.fq.gz       first 2000 read pairs of example/data/NA12878.20slice.30X.fastq.gz (interleaved)
  ex_reads_2k.self.json   SELF-golden (oracle output hashes for those reads): pins GPU == oracle and guards the oracle
                          against accidental change; it does NOT pin oracle == bwa (no bwa exists in the reference tree).
"""
import gzip, hashlib, json, os, subprocess, sys, tempfile
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(os.environ["SPEEDSEQ_CHECKOUT"], "example", "data")
FA = os.path.join(REF, "human_g1k_v37_20_42220611-42542245.fasta")
FQ = os.path.join(REF, "NA12878.20slice.30X.fastq.gz")


def sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def main():
    with open(FA, "rb") as f, gzip.GzipFile(os.path.join(HERE, "ex_ref.fa.gz"), "wb", mtime=0) as g:
        g.write(f.read())
    idx = {e: {"sha256": sha(FA + "." + e), "size": os.path.getsize(FA + "." + e)} for e in ("amb", "ann", "pac", "bwt", "sa")}
    json.dump(idx, open(os.path.join(HERE, "ex_index.sha256.json"), "w"), indent=1, sort_keys=True)
    with gzip.open(FQ, "rt") as f, gzip.GzipFile(os.path.join(HERE, "ex_reads_2k.fq.gz"), "wb", mtime=0) as g:
        for i, l in enumerate(f):
            if i >= 2000 * 2 * 4:
                break
            g.write(l.encode())
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    with tempfile.TemporaryDirectory() as d:
        fa = os.path.join(d, "ex.fa")
        open(fa, "wb").write(gzip.open(os.path.join(HERE, "ex_ref.fa.gz")).read())
        ssqo = os.path.join(ROOT, "oracle", "ssqo")
        subprocess.check_call([ssqo, "index", fa])
        sam = subprocess.run([ssqo, "mem", "-t", "1", "-p", "-R", r"@RG\tID:NA12878\tSM:NA12878\tLB:lib1", fa, os.path.join(HERE, "ex_reads_2k.fq.gz")],
                             check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
        body = b"".join(l for l in sam.splitlines(True) if not l.startswith(b"@PG"))
        sb = subprocess.run([ssqo, "samblaster", "--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20",
                             "--splitterFile", os.path.join(d, "spl.sam"), "--discordantFile", os.path.join(d, "disc.sam")],
                            input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
        strip = lambda b: b"".join(l for l in b.splitlines(True) if not l.startswith(b"@PG"))
        self_golden = {
            "note": "oracle self-golden; NOT a reference known-answer",
            "bwa_mem_sam_sha256_without_PG": hashlib.sha256(body).hexdigest(),
            "samblaster_sam_sha256_without_PG": hashlib.sha256(strip(sb)).hexdigest(),
            "splitters_sha256_without_PG": hashlib.sha256(strip(open(os.path.join(d, "spl.sam"), "rb").read())).hexdigest(),
            "discordants_sha256_without_PG": hashlib.sha256(strip(open(os.path.join(d, "disc.sam"), "rb").read())).hexdigest(),
            "n_sam_lines": body.count(b"\n"),
        }
        json.dump(self_golden, open(os.path.join(HERE, "ex_reads_2k.self.json"), "w"), indent=1, sort_keys=True)
    print("wrote fixtures to", HERE)


if __name__ == "__main__":
    sys.exit(main())
