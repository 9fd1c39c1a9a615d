#!/bin/bash
# ablation of the tensor-core log-likelihood kernel: which stage bounds it
# bits: 1 no global stores, 4 no MMAs, 8 no epilogue work, 16 no prototype TMA loads
for d in ${@:-0 1 4 8 12 20 28}; do
  MGP_TC_DEBUG=$d ncu --metrics gpu__time_duration.sum --clock-control none --csv -k regex:logprob_tc_kernel -s 1 -c 1 python tools/prof_logprob.py tc 0 2 2>/dev/null | grep logprob_tc | rev | cut -d, -f1 | rev | sed "s/^/debug=$d  ns=/"
done
