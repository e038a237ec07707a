#!/bin/bash
# oracle/make_data.sh -- stage the reference-comparison test DATA under
# oracle/_ref/data/ (git-ignored, beside the reference binaries that the tests
# using it run): the reference's bundled
# example index / FASTA / reads (data files, not sources), the linear
# 22_20-21M index built with the reference's own hisat2-build-s (index
# construction is out of scope, SURVEY.md section 2), and seeded synthetic reads.
set -e
cd "$(dirname "$0")"
REF=${REF:-/root/reference}
D=_ref/data
mkdir -p $D
cp --update=none $REF/example/index/22_20-21M_snp.*.ht2 $D/
cp --update=none $REF/example/reference/22_20-21M.fa $REF/example/reference/22_20-21M.snp $D/
cp --update=none $REF/example/reads/reads_1.fa $REF/example/reads/reads_2.fa $D/
if [ ! -f $D/22_20-21M.1.ht2 ]; then
  ./_ref/hisat2-build-s -q $D/22_20-21M.fa $D/22_20-21M > /dev/null
fi
chmod u+w $D/*
if [ ! -f $D/sim10k_1.fa ]; then
  python ../tools/simreads.py $D/22_20-21M.fa 10000 $D/sim10k --seed 1 --paired
fi
if [ ! -f $D/hard20k_1.fa ]; then
  python ../tools/simreads.py $D/22_20-21M.fa 20000 $D/hard20k --seed 3 --paired --indel 0.004 --nrate 0.003 --sub 0.02 --ragged
fi
# short (36 bp: ragged down to empty / 1-3 base reads) and long (150, 250 bp) reads, with indels and Ns
for L in 36 150 250; do
  if [ ! -f $D/len${L}_1.fa ]; then
    python ../tools/simreads.py $D/22_20-21M.fa 20000 $D/len${L} --seed $((70 + L)) --paired --indel 0.004 --nrate 0.002 --sub 0.01 --ragged --rdlen $L
  fi
done
# long reads (the capacity is 1 024 bases): 500 and 1000 bp, 3 000 pairs each
for L in 500 1000; do
  if [ ! -f $D/len${L}_1.fa ]; then
    python ../tools/simreads.py $D/22_20-21M.fa 3000 $D/len${L} --seed $((70 + L)) --paired --indel 0.003 --nrate 0.002 --sub 0.01 --ragged --rdlen $L
  fi
done
# reads carrying ALT alleles of the bundled SNP list (graph index 22_20-21M_snp)
if [ ! -f $D/alt20k_1.fa ]; then
  python ../tools/altreads.py $D/22_20-21M.fa $D/22_20-21M.snp 20000 $D/alt20k --seed 9 --paired
fi
if [ ! -f $D/sim200k_1.fa ]; then
  python ../tools/simreads.py $D/22_20-21M.fa 200000 $D/sim200k --seed 5 --paired
fi
