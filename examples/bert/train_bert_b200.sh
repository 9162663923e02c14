#!/usr/bin/env bash
# Single node, one process per H100, gradient all-reduce on the NVLink peer-memory kernels.
# usage: bash examples/bert/train_bert_b200.sh <data-dir> [save-dir]
set -euo pipefail
DATA=${1:?data directory with dict.txt, train.lmdb, valid.lmdb}
SAVE=${2:-./save/bert_base}
NGPU=${NGPU:-$(nvidia-smi -L | wc -l)}
PORT=${MASTER_PORT:-10086}
export NCCL_ASYNC_ERROR_HANDLING=1
export OMP_NUM_THREADS=${OMP_NUM_THREADS:-4}
python -m torch.distributed.run --nnodes=1 --nproc-per-node="$NGPU" --master-addr 127.0.0.1 --master-port "$PORT" \
    "$(dirname "$0")/../../unicore_cli/train.py" "$DATA" --user-dir "$(dirname "$0")" \
    --train-subset train --valid-subset valid --num-workers 8 --ddp-backend b200 --pin-memory \
    --task bert --loss masked_lm --arch bert_base \
    --optimizer adam --adam-betas "(0.9, 0.98)" --adam-eps 1e-6 --clip-norm 1.0 --weight-decay 1e-4 \
    --lr-scheduler polynomial_decay --lr 1e-4 --warmup-updates 10000 --total-num-update 1000000 \
    --max-update 1000000 --update-freq 1 --batch-size 32 --max-seq-len 512 \
    --fp16 --fp16-init-scale 4 --fp16-scale-window 256 --seed 1 \
    --log-interval 100 --log-format simple --save-interval-updates 10000 --validate-interval-updates 10000 \
    --keep-interval-updates 10 --no-epoch-checkpoints --save-dir "$SAVE" --tmp-save-dir "$SAVE/tmp"
