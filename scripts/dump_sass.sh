#!/bin/bash
# Writes the SASS listings of the compositors and of the stratum sort (the kernels the round-2 review asked for) to
# profiles/sass/, plus a mnemonic histogram of every kernel of the library.  Usage: bash scripts/dump_sass.sh
cd "$(dirname "$0")/.."
mkdir -p profiles/sass
dump() {  # object file, substring of the mangled name, output name
  f=$(cuobjdump -sass pf3plat_b200/csrc/$1.o | grep "Function :" | sed 's/.*Function : //' | grep "$2" | head -1)
  cuobjdump -sass -fun "$f" pf3plat_b200/csrc/$1.o | grep -v "^Fatbin\|^=====\|^arch\|^code version\|^host\|^compile_size\|^$" | sed 's/ *\/\* 0x[0-9a-f]* \*\/$//' > profiles/sass/$3.sass
  echo "$3: $(grep -cE '^\s+/\*[0-9a-f]{4}\*/' profiles/sass/$3.sass) instructions"
}
dump gs_composite_fwd "k_composite_fwd_wsILb0" r2_k_composite_fwd_warp_specialised
dump gs_composite_fwd "15k_composite_fwdILb0" r2_k_composite_fwd_v1
dump gs_composite_bwd "k_composite_bwdILb0ELi256" r2_k_composite_bwd_pair_matrix
dump gs_composite_bwd "k_composite_bwd_v1ILb0" r2_k_composite_bwd_v1
dump gs_binning "k_stratum_rank_sort" r2_k_stratum_rank_sort
dump gs_preprocess "k_sh_colour" r2_k_sh_colour
# (the per-kernel mnemonic histogram profiles/r2_sass_mnemonics.txt is written by scripts/sass_mnemonics.py)
dump gs_lpips "k_conv3x3" lpips_k_conv3x3   # tensor cores: HMMA.1688.F32.TF32
