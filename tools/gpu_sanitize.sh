#!/bin/bash
# compute-sanitizer over one small exec of every kernel family (tests/sanitize_check.py), of every overlap-save convolution
# variant (tests/sanitize_conv_check.py), of every 2-D real transform variant (tests/sanitize_real2d_check.py), of every 2-D
# convolution kernel (tests/sanitize_conv2d_check.py), of every DCT / DST kernel (tests/sanitize_dct_check.py), of every STFT kernel
# (tests/sanitize_stft_check.py), of the chirp-z transform kernels (tests/sanitize_czt_check.py), of the 3-D plans' axis pass
# (tests/sanitize_fft3d_check.py), of every multi-channel convolution variant (tests/sanitize_chconv_check.py), of the
# analytic-signal kernels (tests/sanitize_hilbert_check.py) and of the MDCT kernels (tests/sanitize_mdct_check.py); logs summarised
# in $OUT/summary.txt.
#   default build/switches: memcheck, racecheck, synccheck;  chunked two-pass (B200FFT_FUSED=0): racecheck;
#   dataflow kernel (B200FFT_FLOW=1): memcheck;  TMA-pipelined one-pass kernels (B200FFT_PIPELINE=1): racecheck
OUT=${1:-${TMPDIR:-/tmp}/b200fft_sanitize}
LIMIT=${2:-170}
mkdir -p $OUT
export PYTHONPATH=$PWD:$PWD/tests
CS=/usr/local/cuda/bin/compute-sanitizer
run() {  # name tool env...
    runs tests/sanitize_check.py "$@"
}
runs() {  # script name tool env...
    local script=$1 name=$2 tool=$3; shift 3
    ( export "$@" _X=1; timeout $LIMIT $CS --tool $tool --print-limit 20 --error-exitcode 86 python $script > $OUT/$name.log 2>&1; echo "rc=$?" >> $OUT/$name.log )
    echo "== $name: $(grep -c '^ok' $OUT/$name.log) execs ok, $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|rc=' $OUT/$name.log | tr '\n' ' ')"
}
run default_memcheck memcheck
run default_racecheck racecheck
run default_synccheck synccheck
runs tests/sanitize_conv_check.py conv_memcheck memcheck
runs tests/sanitize_conv_check.py conv_racecheck racecheck
runs tests/sanitize_real2d_check.py real2d_memcheck memcheck
runs tests/sanitize_real2d_check.py real2d_racecheck racecheck
runs tests/sanitize_conv2d_check.py conv2d_memcheck memcheck
runs tests/sanitize_conv2d_check.py conv2d_racecheck racecheck
runs tests/sanitize_dct_check.py dct_memcheck memcheck
runs tests/sanitize_dct_check.py dct_racecheck racecheck
runs tests/sanitize_dct_check.py dct_synccheck synccheck
runs tests/sanitize_stft_check.py stft_memcheck memcheck
runs tests/sanitize_stft_check.py stft_racecheck racecheck
runs tests/sanitize_stft_check.py stft_synccheck synccheck
runs tests/sanitize_czt_check.py czt_memcheck memcheck
runs tests/sanitize_czt_check.py czt_racecheck racecheck
runs tests/sanitize_czt_check.py czt_synccheck synccheck
runs tests/sanitize_fft3d_check.py fft3d_memcheck memcheck
runs tests/sanitize_fft3d_check.py fft3d_racecheck racecheck
runs tests/sanitize_fft3d_check.py fft3d_synccheck synccheck
runs tests/sanitize_chconv_check.py chconv_memcheck memcheck
runs tests/sanitize_chconv_check.py chconv_racecheck racecheck
runs tests/sanitize_chconv_check.py chconv_synccheck synccheck
runs tests/sanitize_hilbert_check.py hilbert_memcheck memcheck
runs tests/sanitize_hilbert_check.py hilbert_racecheck racecheck
runs tests/sanitize_hilbert_check.py hilbert_synccheck synccheck
runs tests/sanitize_mdct_check.py mdct_memcheck memcheck
runs tests/sanitize_mdct_check.py mdct_racecheck racecheck
runs tests/sanitize_mdct_check.py mdct_synccheck synccheck
if [ -z "$SANITIZE_DEFAULT_ONLY" ]; then
run chunked_racecheck racecheck B200FFT_FUSED=0 SANITIZE_QUICK=1
run flow_memcheck memcheck B200FFT_FLOW=1 SANITIZE_QUICK=1
run pipelined_racecheck racecheck B200FFT_PIPELINE=1 SANITIZE_QUICK=1
fi
for f in $OUT/*.log; do echo "--- $f"; grep -E "^ok|SUMMARY|rc=|Error|error|Race|Hazard" $f | head -60; done > $OUT/summary.txt
