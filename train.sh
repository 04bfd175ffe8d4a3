#!/bin/sh
# 1 GPU:  sh train.sh            8 GPUs (data parallel): NPROC=8 sh train.sh
# EVAL_STEPS=k: evaluate the held-out sets of DATA_DIR every k steps (<MODEL_PATH>.eval.jsonl)
# EVAL_SETS: which sets (default in_test,out_test as preprocess.py writes them; dev,test for preprocess_libri.py)
NPROC=${NPROC:-1}
python -m torch.distributed.run --standalone --local-addr 127.0.0.1 --nproc-per-node "$NPROC" main.py \
    -c config.yaml -d "${DATA_DIR:-synthetic}" -train_set train_128 -train_index_file train_samples_128.json \
    -store_model_path "${MODEL_PATH:-vctk_model}" -t vctk_model -iters "${ITERS:-500000}" -summary_steps 500 \
    -eval_steps "${EVAL_STEPS:-0}" -eval_sets "${EVAL_SETS:-in_test,out_test}"
