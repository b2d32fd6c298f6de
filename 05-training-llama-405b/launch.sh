#!/bin/bash
# Launch chapter 05 on every host of ./hosts (one tmux session per node, 8 ranks each) through ssh.
#   bash launch.sh [experiment-name]
# Monitor with:  python ../top-cluster.py hosts      Kill with:  xargs -a hosts -I{} ssh {} tmux kill-session -t dtg-405b
set -euo pipefail
EXPERIMENT_NAME=${1:-llama-405b}
HOSTS_FILE=$(dirname "$0")/hosts
HEAD=$(head -n 1 "$HOSTS_FILE")
NNODES=$(grep -c . "$HOSTS_FILE")
WORKDIR=$(cd "$(dirname "$0")" && pwd)

REMOTE_CMD="cd $WORKDIR && \
  export OMP_NUM_THREADS=26 TORCH_NCCL_AVOID_RECORD_STREAMS=1 NCCL_CROSS_NIC=1 && \
  export TORCHELASTIC_ERROR_FILE=../error.json && \
  python -m torch.distributed.run \
    --rdzv-id $EXPERIMENT_NAME --rdzv-backend c10d --rdzv-endpoint $HEAD:5001 \
    --nnodes $NNODES --nproc-per-node gpu --redirects 3 --log-dir ../logs \
    train_llm.py \
      --experiment-name $EXPERIMENT_NAME \
      --dataset-name Skylion007/openwebtext \
      --model-name meta-llama/Llama-3.1-405B \
      --batch-size 1 --seq-length 2048 \
      --cpu-offload --checkpoint-activations --prefetch-layers --log-freq 1"

xargs -a "$HOSTS_FILE" -I {} ssh {} tmux new-session -d -s dtg-405b "bash -lc '$REMOTE_CMD'"
echo "started on $NNODES nodes; logs under ../logs, attach with: ssh $HEAD tmux attach -t dtg-405b"
