#!/usr/bin/env bash
# One command that produces an ncu capture for every kernel family of libkge_b200.  Run from the repo root on ONE GPU
# (ncu replays each kernel ~40x):
#   bash scripts/ncu_all.sh <tag> [capture names]
# Outputs (small CSV/JSON summaries, no .ncu-rep) land in $NCU_OUT (default ncu_out/, ignored by git).
set -uo pipefail
tag=${1:-rX}
only=${2:-all}   # 'all', or a space-separated list of capture names to run (e.g. "train_cfg3 train_cfg4 rank_rotate")
out=${NCU_OUT:-ncu_out}
mkdir -p $out
NCU="ncu --clock-control none"

want() { [ "$only" = all ] || [[ " $only " == *" $1 "* ]]; }
cap() {  # cap <name> <kernel regex> <skip> <count> <cmd...>
  local name=$1 regex=$2 skip=$3 count=$4; shift 4
  want "$name" || return 0
  timeout 400 $NCU --set full --import-source on -k "regex:$regex" -s "$skip" -c "$count" -f -o "$out/${tag}_$name" "$@" > "$out/${tag}_$name.stdout" 2>&1
  ncu -i "$out/${tag}_$name.ncu-rep" --page raw --csv > "$out/${tag}_${name}_raw.csv" 2>/dev/null
  python scripts/ncu_summary.py full "$out/${tag}_${name}_raw.csv" "$out/${tag}_${name}_ncu_full_summary.json" \
      "ncu --set full --clock-control none --import-source on -k regex:$regex -s $skip -c $count $*"
  rm -f "$out/${tag}_$name.ncu-rep" "$out/${tag}_${name}_raw.csv"
}
launches() {  # launches <name> <count> <cmd...>
  local name=$1 count=$2; shift 2
  want "launches_$name" || return 0
  timeout 400 $NCU --metrics gpu__time_duration.sum -c "$count" --csv --log-file "$out/${tag}_launches_$name.csv" "$@" > /dev/null 2>&1
  python scripts/ncu_summary.py launches "$out/${tag}_launches_$name.csv" "$out/${tag}_launch_list_${name}_summary.csv" \
      "ncu --metrics gpu__time_duration.sum --clock-control none -c $count $*"
}

# launch lists: the bench step (kernel shares of a training step) and one evaluate call (kernel shares of kge_rank)
launches bench 300 python bench.py --steps 5 --warmup 3 --no-cpu --no-extra
launches evaluate 200 python scripts/rbench.py one ComplEx 200 14505 1024

# training kernels: resident ComplEx (cfg2, fast path), resident DistMult NIT=4 (cfg3, fast path), RotatE fast path (cfg4), HBM-resident table
# (big: resident geometry, 3.2 GB table), windowed + grouped ComplEx k=1000 (cfg5w: 1.6 GB table)
cap train_cfg2 'kge_train_res_kernel|kge_optim_kernel' 8 2 python bench.py --steps 5 --warmup 3 --no-cpu --no-extra
cap train_cfg3 kge_train_res_kernel 2 1 python scripts/kbench.py one cfg3 0
cap train_cfg4 kge_train_rot_kernel 2 1 python scripts/kbench.py one cfg4 0
cap train_big  kge_train_res_kernel 2 1 python scripts/kbench.py one big 0
cap train_cfg5w kge_train_kernel 2 1 python scripts/kbench.py one cfg5w 0
# optimizers: lazy (touched rows only) and the one-launch exchange kernel (world = 1: a multi-rank command must not run under ncu)
cap optim_lazy kge_optim_lazy_kernel 2 1 python -m pytest tests/test_gpu_parity.py -q -k "lazy_optimizer_matches_restatement and lazy_adam"
cap optim_exchange kge_optim_exchange_kernel 1 1 python -m pytest tests/test_gpu_parity.py -q -k exchange_kernel_world1
# ranking kernels: tensor-core filter + its helpers (ComplEx, auto mode), FP32 dot kernel (exact mode), pair kernel (TransE, RotatE)
cap rank_tc 'kge_rank_tc_kernel|kge_rank_split_kernel|kge_rank_refine_kernel' 0 8 python scripts/rbench.py one ComplEx 200 14505 1024
KGE_B200_RANK_MODE=exact cap rank_dot 'kge_rank_dot_kernel|kge_rank_q|kge_rank_finalize' 0 4 python scripts/rbench.py one ComplEx 200 14505 1024
cap rank_transe kge_rank_pair_kernel 0 1 python scripts/rbench.py one TransE 400 14505 1024
cap rank_rotate kge_rank_pair_kernel 0 2 python scripts/rbench.py one RotatE 200 14505 1024
ls -la $out | tail -30
