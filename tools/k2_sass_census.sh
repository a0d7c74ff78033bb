#!/bin/bash
# Static instruction census of K2's window loop; needs no GPU. Runs tools/k1_sass_census.sh on k2_decompress_kernel:
# the kernel's registers and spills from -Xptxas -v, then per loop the instruction count and the instructions that cost
# more than an issue slot (SHFL, VOTE, REDUX, LDS/STS, global LD/ST, BSSY, ...). The loop at depth 0 is a warp's loop
# over its streams, the one at depth 1 the window loop of k2_decode_stream (with its rare blocks: the per-element error
# checks, the serial replay of dependent copies and the spilling literal's copy); the loops nested in it are the
# flattened-copy loop, the replay loop and warp_copy's. WAITS=1 adds the scoreboard table of the window loop: for every
# load, the first instruction that waits on it and the distance. A static count is not a time.
# usage: tools/k2_sass_census.sh [extra nvcc flags]; MIN, WAITS, HEAD and SASS as for k1_sass_census.sh.
# The cubin, the SASS listing and the ptxas log go to $OUT (default build/k2_exp, kept out of git).
cd "$(dirname "$0")/.."
KERNEL=k2_decompress_kernel DEPTH=${DEPTH:-1} MIN=${MIN:-20} OUT=${OUT:-build/k2_exp} exec tools/k1_sass_census.sh "$@"
