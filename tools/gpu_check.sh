#!/bin/bash
# One GPU-box session: every step under its own `timeout -k`, stop at the first step that hangs.
#
#   gpurun --gpus N --timeout S -- 'bash tools/gpu_check.sh [N] [step ...]'
#
# Steps (default: pytest smoke bench ref):
#   pytest  GPU test suite                 smoke  __graft_entry__.smoke()
#   bench   bench.py at N GPUs             ref    bench.py --impl reference at N GPUs
#   quick   bench.py without extras / e2e  lab    bench/r2_lab.py sweeps (1 or 2 GPUs)
#   lat     bench/configs.py latency       ncu    bench/ncu_driver.py under ncu --set full (1 process)
#   fp8     bench/configs.py fp8 (ring)    fanin  bench/configs.py fanin
#   fp8ab   fp8 ring with grid caps 264 / 132 (2 / 1 per H100 SM), twice, interleaved
#
# A step that runs into its limit may have wedged the GPU (it has happened: a multicast bulk
# load from peer memory); going on would burn the whole gpurun limit, so the script aborts.
N=${1:-1}; shift
STEPS=${*:-pytest smoke bench ref}
OUT=gpurun_out; mkdir -p $OUT
step() {
    local name=$1 secs=$2; shift 2
    timeout -k 10 "$secs" "$@" > "$OUT/check_$name.txt" 2> "$OUT/check_$name.err"
    local rc=$?
    echo "== $name rc=$rc"; tail -3 "$OUT/check_$name.txt" | cut -c1-800
    [ $rc -ne 0 ] && tail -5 "$OUT/check_$name.err" | cut -c1-400
    if [ $rc -eq 124 ] || [ $rc -eq 137 ]; then echo "ABORT: $name ran into its limit"; exit 1; fi
}
port=29517
launch() {   # python, or torchrun with N ranks on a fresh port
    if [ "$N" -gt 1 ]; then
        port=$((port + 10))
        LAUNCH="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $port"
    else
        LAUNCH="python"
    fi
}
for s in $STEPS; do
    launch
    case $s in
    pytest) step pytest 600 python -m pytest tests -m gpu -q ;;
    smoke)  step smoke 120 python __graft_entry__.py smoke ;;
    bench)  step bench 600 $LAUNCH bench.py --gpus $N --steps 6 --warmup 3 ;;
    quick)  step quick 300 $LAUNCH bench.py --gpus $N --steps 4 --warmup 3 --no-extra --no-e2e ;;
    ref)    step ref 600 $LAUNCH bench.py --impl reference --gpus $N --steps 3 --warmup 1 ;;
    lat)    step lat 200 $LAUNCH bench/configs.py latency ;;
    fp8)    step fp8 300 $LAUNCH bench/configs.py fp8 ;;
    fp8ab)  for i in 1 2; do for c in 264 132; do   # interleaved A/B of the client's grid cap
                launch; step fp8_ctas${c}_$i 300 $LAUNCH bench/configs.py fp8 --max-ctas $c
            done; done ;;
    fanin)  step fanin 300 $LAUNCH bench/configs.py fanin ;;
    lab)    step lab 600 $LAUNCH bench/r2_lab.py ;;
    ncu)    step ncu 900 ncu --set full --section Nvlink --clock-control none --import-source on \
                -o $OUT/all_kernels -f python bench/ncu_driver.py ;;
    *) echo "unknown step $s" ;;
    esac
done
