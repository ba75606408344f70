#!/bin/bash
# One `ncu --set full` capture per non-LDPC hot-path kernel (run on the GPU box; reports land in gpurun_out/).
set -x
cap() {  # name kernel-regex
  ncu --set full --clock-control none --import-source on -k "regex:$2" -c 1 -f -o gpurun_out/phy_$1 \
      python tools/bench_phy_kernels.py --only $1 > /dev/null 2>&1
}
cap demapper_app_64qam demap_qam_kernel
cap demapper_maxlog_64qam demap_qam_kernel
cap ofdm_demodulate_76 ofdm_fft_small_kernel
cap ofdm_modulate_4096 ofdm_fft_r16_kernel
cap ofdm_lmmse_4x16 ofdm_lmmse_diag_kernel
cap ls_estimator_lin_4x16 interp_lin_kernel
cap ldpc5g_encode_4224_8448 ldpc5g_encode_kernel
ls -la gpurun_out/phy_*.ncu-rep
