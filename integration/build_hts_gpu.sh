#!/bin/bash
# The drop-in, for real: the UNMODIFIED reference (htslib 1.23.1) built against libhtsgpu.so.
#
#   * bgzf.c is compiled with -DHAVE_HTSGPU after integration/htsgpu_bgzf.patch is applied to a
#     scratch copy (the patch is the only thing kept here; no reference source is copied into the
#     repository): bgzf_mt_reader hands batches of bgzf_job to hgpu_bgzf_inflate_jobs_host, the
#     unthreaded inflate_block sends single blocks the same way.
#   * the htscodecs entropy coders (rANS 4x8 / Nx16, arith_dynamic, tok3, fqzcomp) are NOT compiled:
#     cram/cram_io.c resolves rans_uncompress_4x16, tok3_decode_names, ... to libhtsgpu.so, which is
#     what ./configure --with-external-htscodecs (configure.ac:278-282) does with -lhtscodecs.
#     hts_pack / hts_unpack(_meta) / hts_rle_encode / hts_rle_decode / htscodecs_version (bound by cram_codecs.c and
#     cram_external.c) come from libhtsgpu.so as well (xform.cu); only utils.c (thread-local scratch) is compiled from
#     the reference as it stands.
#   * everything else is compiled from /root/reference where it lies, exactly as oracle/build_ref.sh
#     does for the stock build.
#
# Output (git-ignored; under oracle/_ref/ with the stock build, so both travel together):
# oracle/_ref/integration/libhts_gpu.so and the reference's own test programs linked against it:
# test_bgzf, test_view, bgzip (and the same three on the stock build in stock/).
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
ROOT=$(dirname "$HERE")
OUT=${OUT:-$ROOT/oracle/_ref/integration}
[ -d "$REF" ] || { echo "no reference tree at $REF; keeping prebuilt $OUT" >&2; exit 0; }
[ -f "$ROOT/htslib_b200/libhtsgpu.so" ] || { echo "build htslib_b200/libhtsgpu.so first" >&2; exit 1; }
mkdir -p "$OUT/obj" "$OUT/src"
G=$ROOT/oracle/_ref/gen
[ -f "$G/config.h" ] || bash "$ROOT/oracle/build_ref.sh"

# patched bgzf.c in scratch
cp "$REF/bgzf.c" "$OUT/src/bgzf.c"
chmod u+w "$OUT/src/bgzf.c"
patch -s -p0 "$OUT/src/bgzf.c" < "$HERE/htsgpu_bgzf.patch"

CFLAGS="-O2 -g0 -fPIC -fvisibility=default -w -I$G -I$REF -I$REF/htscodecs/htscodecs -I$ROOT/include"
SRCS="kfunc kstring bcf_sr_sort errmod faidx header hfile hts hts_expr hts_os md5 multipart probaln realn regidx region sam sam_mods simd synced_bcf_reader vcf_sweep tbx textutils thread_pool vcf vcfutils
cram/cram_codecs cram/cram_decode cram/cram_encode cram/cram_external cram/cram_index cram/cram_io cram/cram_stats cram/mFILE cram/open_trace_file cram/pooled_alloc cram/string_alloc
htscodecs/htscodecs/utils"
pids=()
OBJS="$OUT/obj/bgzf.o"
gcc $CFLAGS -DHAVE_HTSGPU -I"$REF" -c "$OUT/src/bgzf.c" -o "$OUT/obj/bgzf.o" &
pids+=($!)
for s in $SRCS; do
  o="$OUT/obj/$(echo $s | tr '/' '_').o"
  OBJS="$OBJS $o"
  if [ ! -f "$o" ] || [ "$REF/$s.c" -nt "$o" ]; then
    gcc $CFLAGS -c "$REF/$s.c" -o "$o" &
    pids+=($!)
    if [ ${#pids[@]} -ge 8 ]; then wait "${pids[0]}"; pids=("${pids[@]:1}"); fi
  fi
done
for p in "${pids[@]}"; do wait $p; done
RP='-Wl,-rpath,$ORIGIN/../../../htslib_b200 -Wl,-rpath,$ORIGIN'
gcc -shared -o "$OUT/libhts_gpu.so" $OBJS -L"$ROOT/htslib_b200" -lhtsgpu $RP -lz -lm -lpthread
for t in test/test_bgzf test/test_view bgzip; do
  gcc $CFLAGS -o "$OUT/$(basename $t)" "$REF/$t.c" -L"$OUT" -lhts_gpu -L"$ROOT/htslib_b200" -lhtsgpu $RP -lz -lm -lpthread
done
# the same three programs on the stock build, for side-by-side comparisons
if [ -f "$ROOT/oracle/_ref/libhts_ref.so" ]; then
  mkdir -p "$OUT/stock"
  for t in test/test_bgzf test/test_view bgzip; do
    gcc $CFLAGS -o "$OUT/stock/$(basename $t)" "$REF/$t.c" -L"$ROOT/oracle/_ref" -lhts_ref '-Wl,-rpath,$ORIGIN/../..' -lz -lm -lpthread
  done
fi
echo "built $OUT/libhts_gpu.so"
nm -D "$OUT/libhts_gpu.so" | grep -E " U (rans_|arith_|tok3_|fqz_|hgpu_|hts_pack|hts_unpack|hts_rle_|htscodecs_version)" | awk '{print "  from libhtsgpu.so:", $2}'
