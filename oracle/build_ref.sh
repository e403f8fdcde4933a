#!/usr/bin/env bash
# oracle/build_ref.sh — TEST INFRASTRUCTURE, not product code.
#
# Compiles the reference's own matcher (Xapiand's vendored Xapian 1.5.0,
# /root/reference/src/xapian) from the sources WHERE THEY LIE into oracle/_ref/:
#   oracle/_ref/libxapian_ref.so   the reference Xapian library (api, matcher, weight, backends …)
#   oracle/_ref/gen/               generated headers (error.h via the reference's own perl generator)
# Nothing from /root/reference is copied into the repository; oracle/_ref/ is git-ignored but
# travels to the GPU box with gpurun.  Recipe = SURVEY.md Appendix A (the reference's own CMake
# build is NOT run: it needs libuuid headers, tclsh and GTest which this image lacks).
# Flags follow the reference release flags (CMakeLists.txt:99-104: -std=c++17 -O3 -DNDEBUG).
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${XGM_REFERENCE:-/root/reference}"
R="$REF/src"
O="$HERE/_ref"
JOBS="${JOBS:-$(nproc)}"

if [ ! -d "$R/xapian" ]; then
  echo "build_ref: $R/xapian not present (GPU box?) — keeping prebuilt $O" >&2
  exit 0
fi
# ---- Xapiand's multivalue classes (src/multivalue), on top of the library above ------------------------
# MultipleValueRange (range.cc:351-414), Multi_MultiValueKeyMaker (keymaker.cc:704-757), StringList
# (serialise_list.h, header only) and Xapiand's own sortable_serialise(long double), compiled from the seven
# source files where they lie (+ geospatial/cartesian.cc, whose constructor a header constant needs).  The query-DSL halves of those files (MultipleValueRange::getQuery, GeoKey)
# call into Xapiand's schema / cast / datetime / geospatial code, which is NOT built: those are function
# symbols only, left undefined in the shared object and bound lazily (-z lazy) — nothing on the matching
# path calls them.  Pins SURVEY.md section 8 rows a15 / a16 against the reference's real code.
build_mv() {   # $1 = "" (against libxapian_ref.so) or "_xgm" (against libxapian_ref_xgm.so)
  local MV="$O/libxapiand_mv_ref$1.so"
  if [ -f "$MV" ] && [ "$MV" -nt "$HERE/ref_mv_glue.cc" ] && [ "${FORCE:-0}" != "1" ]; then return 0; fi
  mkdir -p "$O/obj_mv"
  local MVFLAGS="-std=c++17 -O2 -DNDEBUG -fPIC -w -include limits -include cstdint -include functional -I$O/gen -I$R -I$REF"
  local objs=""
  for f in multivalue/range.cc multivalue/keymaker.cc sortable_serialise.cc length.cc exception.cc fmt/format.cc geospatial/cartesian.cc; do
    local o="$O/obj_mv/$(echo "$f" | tr '/' '_' | sed 's/\.cc$/.o/')"
    objs="$objs $o"
    ( if [ ! -f "$o" ] || [ "$R/$f" -nt "$o" ]; then g++ $MVFLAGS -c "$R/$f" -o "$o"; fi ) &
  done
  # our factory functions around those classes (oracle/ref_mv_glue.cc)
  objs="$objs $O/obj_mv/ref_mv_glue.o"
  g++ $MVFLAGS -c "$HERE/ref_mv_glue.cc" -o "$O/obj_mv/ref_mv_glue.o" &
  wait
  g++ -shared -o "$MV" $objs -L"$O" -lxapian_ref$1 -Wl,-z,lazy -Wl,-rpath,'$ORIGIN'
  echo "build_ref: built $MV"
}

# ---- the variant a maintainer would ship: the same library with the xgm shim at the Matcher::get_mset seam ----
# xapiand_b200/shim/xgm_shim.{h,cc} (ours) + ONE patched line of src/xapian/matcher/matcher.cc (:595, the call of
# get_local_mset): the patched copy is generated with sed into oracle/_ref/gen/ (git-ignored), the reference
# sources stay where they lie.  Every other object file is shared with libxapian_ref.so.
build_xgm() {
  local X="$O/libxapian_ref_xgm.so"
  local SH="$HERE/../xapiand_b200/shim"
  if [ -f "$X" ] && [ "$X" -nt "$SH/xgm_shim.cc" ] && [ "$X" -nt "$SH/xgm_shim.h" ] && [ "$X" -nt "$HERE/../include/xgm.h" ] && [ "${FORCE:-0}" != "1" ]; then
    build_mv _xgm; return 0
  fi
  local XFLAGS="-std=c++17 -O3 -DNDEBUG -fPIC -w -include limits -include cstdint -I$O/gen -I$R -I$R/xapian -I$SH"
  sed -e 's|^#include "xapian/matcher/matcher.h"$|#include "xapian/matcher/matcher.h"\n#include "xgm_shim.h"|' \
      -e 's|local_mset = get_local_mset(first, maxitems, check_at_least,|if (!XGM_SHIM_TRY_LOCAL_MSET(local_mset)) local_mset = get_local_mset(first, maxitems, check_at_least,|' \
      "$R/xapian/matcher/matcher.cc" > "$O/gen/matcher_xgm.cc"
  grep -q XGM_SHIM_TRY_LOCAL_MSET "$O/gen/matcher_xgm.cc" || { echo "build_ref: seam not found in matcher.cc" >&2; exit 1; }
  g++ $XFLAGS -I"$R/xapian/matcher" -c "$O/gen/matcher_xgm.cc" -o "$O/obj/xgm_matcher.o" &
  g++ $XFLAGS -c "$SH/xgm_shim.cc" -o "$O/obj/xgm_shim.o" &
  wait
  g++ -shared -o "$X" $(awk '{print $2}' "$O/obj/.list" | grep -v 'xapian_matcher_matcher\.o$') "$O/obj/xgm_matcher.o" "$O/obj/xgm_shim.o" -lz -lpthread -ldl
  echo "build_ref: built $X"
  build_mv _xgm
}

# a changed build configuration invalidates every object built under the old one
if [ -f "$O/libxapian_ref.so" ] && { [ "$HERE/ref_config.h" -nt "$O/libxapian_ref.so" ] || [ "$HERE/ref_uuid.h" -nt "$O/libxapian_ref.so" ]; }; then
  rm -rf "$O"
fi

if [ -f "$O/libxapian_ref.so" ] && [ "${FORCE:-0}" != "1" ]; then
  echo "build_ref: $O/libxapian_ref.so already built (FORCE=1 to rebuild)"
  build_mv ""
  build_xgm
  exit 0
fi

mkdir -p "$O/gen/xapian/unicode" "$O/gen/xapian/languages" "$O/gen/uuid" "$O/obj"
cp "$HERE/ref_config.h" "$O/gen/config.h"
cp "$HERE/ref_uuid.h" "$O/gen/uuid/uuid.h"
# generated headers, by the reference's own generators (CMakeLists.txt:402-412, 472-479)
(cd "$O/gen" && perl -w -I "$R/xapian" "$R/xapian/generate-exceptions")
perl "$R/xapian/unicode/gen_c_istab" "$O/gen/xapian/unicode/c_istab.h"
printf '#define LANGSTRING "none"\n' > "$O/gen/xapian/languages/sbl-dispatch.h"

# link-only stubs for symbols that live in parts of Xapian needing tclsh/lemon/snowball outputs
# (queryparser, languages, unicode-data); never reached by matching.
cat > "$O/gen/ref_stubs.cc" <<'STUB'
#include "config.h"
#include <cstdlib>
#include <string>
#include "xapian.h"
#include "xapian/api/msetinternal.h"
namespace Xapian {
RangeProcessor::~RangeProcessor() {}
Stem::Stem(const Stem& o) : internal(o.internal) {}
Stem::~Stem() {}
std::string Stem::operator()(const std::string& w) const { return w; }
std::string Stopper::get_description() const { return "Stopper"; }
std::string MSet::Internal::snippet(const std::string&, size_t, const Stem&, unsigned,
                                    const std::string&, const std::string&, const std::string&) const { abort(); }
}
STUB

DIRS="api matcher weight common backends backends/glass backends/inmemory backends/multi backends/honey backends/remote net expand geospatial diversify cluster"
FILES=""
for d in $DIRS; do FILES="$FILES $(ls "$R"/xapian/$d/*.cc)"; done
FILES="$FILES $R/xapian/unicode/description_append.cc $R/xapian/unicode/utf8itor.cc $O/gen/ref_stubs.cc"

CXXFLAGS="-std=c++17 -O3 -DNDEBUG -fPIC -w -include limits -include cstdint -I$O/gen -I$R"
: > "$O/obj/.list"
for f in $FILES; do
  o="$O/obj/$(echo "${f#$R/}" | tr '/' '_' | sed 's/\.cc$/.o/')"
  echo "$f $o" >> "$O/obj/.list"
done
# compile in parallel
xargs -P "$JOBS" -L 1 bash -c 'if [ ! -f "$1" ] || [ "$0" -nt "$1" ]; then g++ '"$CXXFLAGS"' -c "$0" -o "$1" || exit 255; fi' < "$O/obj/.list"
g++ -shared -o "$O/libxapian_ref.so" $(awk '{print $2}' "$O/obj/.list") -lz -lpthread
echo "build_ref: built $O/libxapian_ref.so ($(wc -l < "$O/obj/.list") objects)"
build_mv ""
build_xgm
