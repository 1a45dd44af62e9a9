#!/bin/bash
# Compiles the reference's own stereo-input functions (sources under /root/reference, never copied) into
# oracle/_ref/libinputref.so, which tests/test_stereo_input_oracle.py runs against oracle/input_oracle.c. Outputs go only to
# oracle/_ref/ (git-ignored). Called by __graft_entry__.build(); without the reference tree it keeps what is there.
# No contraction / fast-math, so the reference code is evaluated in plain IEEE binary32.
set -e
REF=${REF:-/root/reference/src/InfiniTAM/InfiniTAM}
DS=${DS:-/root/reference/src/DynSLAM}
HERE="$(cd "$(dirname "$0")" && pwd)"
if [ ! -f "$DS/DepthProvider.h" ] || [ ! -d "$REF/ITMLib" ]; then echo "reference not present; keeping prebuilt oracle/_ref" >&2; exit 0; fi
mkdir -p "$HERE/_ref"

# ---- DynSLAM's stored stereo input: DepthProvider, PrecomputedDepthProvider's conversion and clamp, CvToItm (oracle/_ref/libinputref.so)
# DepthProvider.h, PrecomputedDepthProvider.cpp and InfiniTamDriver.cpp need OpenCV, Pangolin, gflags and the Input pipeline as
# translation units; the class and the three function bodies only need DS/Utils.h's standard headers, OpenCV's matrices
# (oracle/input_stubs) and ORUtils' image. They are cut out of the reference files here, at build time, into oracle/_ref/ (git-ignored)
# and compiled unmodified around oracle/ref_input_driver.cpp.
DPH="$DS/DepthProvider.h"; PDP="$DS/PrecomputedDepthProvider.cpp"; ITD="$DS/InfiniTamDriver.cpp"
if [ -f "$DPH" ] && [ -f "$PDP" ] && [ -f "$ITD" ]; then
  awk '/^struct StereoCalibration \{/ {on=1} on {print} on && /^};$/ && seen {exit} /^class DepthProvider \{/ {seen=1}' "$DPH" > "$HERE/_ref/depthprovider_extract.inc"
  awk '/^  if \(this->input_is_depth_\) \{/ {on=1} on {print} on && /^  }$/ {exit}' "$PDP" > "$HERE/_ref/clamp_extract.inc"
  awk '/^float PrecomputedDepthProvider::DepthFromDisparity\(/ {on=1} on {print} on && /^}$/ {exit}' "$PDP" > "$HERE/_ref/dfd_extract.inc"
  awk '/^void CvToItm\(const cv::Mat3b &/ {on=1} on {print} on && /^}$/ {exit}' "$ITD" > "$HERE/_ref/cvtoitm_extract.inc"
  if grep -q "DepthFromDisparityMap" "$HERE/_ref/depthprovider_extract.inc" && grep -q "max_depth_mm_s" "$HERE/_ref/clamp_extract.inc" && \
     grep -q "DepthFromDisparity" "$HERE/_ref/dfd_extract.inc" && grep -q "255u" "$HERE/_ref/cvtoitm_extract.inc"; then
    /usr/bin/g++ -std=c++14 -O2 -ffp-contract=off -fno-fast-math -shared -fPIC -w -DCOMPILE_WITHOUT_CUDA -I"$HERE/input_stubs" -I"$REF" -I"$HERE" \
        -o "$HERE/_ref/libinputref.so" "$HERE/ref_input_driver.cpp" && echo "built $HERE/_ref/libinputref.so"
  else
    echo "could not locate DepthProvider / PrecomputedDepthProvider / CvToItm in $DS" >&2
  fi
  rm -f "$HERE/_ref/depthprovider_extract.inc" "$HERE/_ref/clamp_extract.inc" "$HERE/_ref/dfd_extract.inc" "$HERE/_ref/cvtoitm_extract.inc"
fi
