# Multi-GPU evidence run (on a machine with 8 GPUs): NCCL DP test on 2 ranks, then the default bench line under torchrun at the N given
# in $SCALE_NS (default "8 2").
set -x
mkdir -p gpurun_out
timeout 300 python -m pytest tests/test_gpu_dp.py -m gpu -x -q > gpurun_out/r02_dp_test.log 2>&1; tail -5 gpurun_out/r02_dp_test.log
for N in ${SCALE_NS:-8 2}; do
  timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $((29600+N)) bench.py --gpus $N --steps 20 --warmup 5 --no-cpu-baseline > gpurun_out/r02_scale_n$N.json 2> gpurun_out/r02_scale_n$N.err
done
python - <<'PY'
import json
for N in (1,2,4,8):
    try:
        d=json.loads(open(f'gpurun_out/r02_scale_n{N}.json').read().strip().splitlines()[-1]); t=d['train']
        print(N, 'infer M frames/s', round(d['value']/1e6,2), 'ms', round(d['ms_per_step'],3), 'e2e', round(d['e2e']['value']/1e6,2), '| train steps/s', round(t['value'],2), 'ms', round(t['ms_per_step'],3), 'exposed', round(t['nccl_exposed_ms'],3), 'e2e', round(t['e2e']['value'],2), 'clocks', d['clocks']['reasons'])
    except Exception as e: print(N, e)
PY
