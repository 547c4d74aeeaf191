#!/bin/bash
# Build the UNMODIFIED reference (htslib 1.23.1 + htscodecs 1.6.6) from the sources where
# they lie under /root/reference into oracle/_ref/ (git-ignored; travels to the GPU box).
# This is TEST INFRASTRUCTURE (the parity checker and the CPU baseline), never the product.
# We do not run the reference's build system: plain gcc on its .c files with a generated
# config.h equal to what Makefile:303-350 would write minus the libraries absent here
# (bz2, lzma, curl; zlib arm of bgzf.c since libdeflate is absent).
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
[ -d "$REF" ] || { echo "no reference tree at $REF; keeping prebuilt $OUT" >&2; exit 0; }
mkdir -p "$OUT/gen" "$OUT/obj"
G=$OUT/gen
cat > "$G/config.h" <<'EOC'
/* config.h for the oracle build: Makefile default minus bz2/lzma/curl */
#ifndef _XOPEN_SOURCE
#define _XOPEN_SOURCE 600
#endif
#define HAVE_DRAND48 1
#if defined __x86_64__
#define HAVE_DECL___CPUID_COUNT 1
#define HAVE_DECL___GET_CPUID_MAX 1
#define HAVE_POPCNT 1
#define HAVE_SSE4_1 1
#define HAVE_SSSE3 1
#define HAVE_AVX2 1
#define HAVE_AVX512 1
#define HAVE_X86INTRIN_H 1
#define HAVE_ATTRIBUTE_TARGET_SSSE3 1
#define HAVE_BUILTIN_CPU_SUPPORT_SSSE3 1
#endif
#if defined __x86_64__ || defined __arm__ || defined __aarch64__
#define HAVE_ATTRIBUTE_CONSTRUCTOR 1
#endif
#if defined __linux__
#define HAVE_GETAUXVAL
#endif
EOC
printf '#define HTS_VERSION_TEXT "1.23.1"\n#define HTSCODECS_VERSION_TEXT "1.6.6"\n' > "$G/version.h"
printf '#define HTS_CC "gcc"\n#define HTS_CPPFLAGS ""\n#define HTS_CFLAGS "-O2"\n#define HTS_LDFLAGS ""\n#define HTS_LIBS "-lz -lm -lpthread"\n' > "$G/config_vars.h"

CFLAGS="-O2 -g0 -fPIC -fvisibility=default -w -I$G -I$REF -I$REF/htscodecs/htscodecs"
SRCS="kfunc kstring bcf_sr_sort bgzf errmod faidx header hfile hts hts_expr hts_os md5 multipart probaln realn regidx region sam sam_mods simd synced_bcf_reader vcf_sweep tbx textutils thread_pool vcf vcfutils
cram/cram_codecs cram/cram_decode cram/cram_encode cram/cram_external cram/cram_index cram/cram_io cram/cram_stats cram/mFILE cram/open_trace_file cram/pooled_alloc cram/string_alloc
htscodecs/htscodecs/arith_dynamic htscodecs/htscodecs/fqzcomp_qual htscodecs/htscodecs/htscodecs htscodecs/htscodecs/pack htscodecs/htscodecs/rANS_static4x16pr htscodecs/htscodecs/rANS_static32x16pr htscodecs/htscodecs/rANS_static htscodecs/htscodecs/rle htscodecs/htscodecs/tokenise_name3 htscodecs/htscodecs/utils
htscodecs/htscodecs/rANS_static32x16pr_avx2 htscodecs/htscodecs/rANS_static32x16pr_avx512 htscodecs/htscodecs/rANS_static32x16pr_sse4 htscodecs/htscodecs/rANS_static32x16pr_neon"
pids=()
OBJS=""
for s in $SRCS; do
  o="$OUT/obj/$(echo $s | tr '/' '_').o"
  OBJS="$OBJS $o"
  extra=""
  case "$s" in
    *_avx2)   extra="-mavx2 -mpopcnt" ;;
    *_avx512) extra="-mavx512f -mpopcnt" ;;
    *_sse4)   extra="-msse4.1 -mssse3 -mpopcnt" ;;
  esac
  if [ ! -f "$o" ] || [ "$REF/$s.c" -nt "$o" ]; then
    gcc $CFLAGS $extra -c "$REF/$s.c" -o "$o" &
    pids+=($!)
    if [ ${#pids[@]} -ge 8 ]; then wait "${pids[0]}"; pids=("${pids[@]:1}"); fi
  fi
done
for p in "${pids[@]}"; do wait $p; done
gcc -shared -o "$OUT/libhts_ref.so" $OBJS -lz -lm -lpthread
echo "built $OUT/libhts_ref.so"
# the reference's own test programs around libhtsgpu.so (tests/test_integration.py), once the product is built
if [ -f "$HERE/../htslib_b200/libhtsgpu.so" ]; then
  bash "$HERE/../integration/build_hts_gpu.sh"
fi
