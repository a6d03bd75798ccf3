#!/usr/bin/env bash
# Accuracy benchmark (counterpart of reference benchmarks/accuracy/run.sh): train the same model with the sm_90a
# kernels and with the plain-PyTorch reference ops, then assert |delta train_loss| <= 1e-2.
#   NPROC=1 MODEL=llama3.2-1b STEPS=200 bash benchmarks/accuracy/run.sh
#   HF=1 ...      the HuggingFace LlamaForCausalLM of the same geometry through ta.accelerate (the object the reference's
#                 protocol wraps); SP=2 NPROC=2 ... adds Ulysses context parallelism
set -euo pipefail
cd "$(dirname "$0")/../.."
NPROC=${NPROC:-1}; MODEL=${MODEL:-llama3.2-1b}; STEPS=${STEPS:-200}; SEQ=${SEQ:-1024}; BS=${BS:-4}
OUT=${OUT:-log/accuracy}; mkdir -p "$OUT"
LAUNCH="python"
if [ "$NPROC" -gt 1 ]; then
  LAUNCH="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NPROC --master-addr 127.0.0.1 --master-port ${PORT:-29671}"
fi
for impl in torch native; do
  $LAUNCH benchmarks/accuracy/run_clm.py --impl $impl --model "$MODEL" --steps "$STEPS" --seq_len "$SEQ" \
      --batch_size "$BS" ${LAYERS:+--layers $LAYERS} ${HF:+--hf} ${SP:+--sp_size $SP} --out "$OUT/$impl.json" 2>&1 | tee "$OUT/$impl.log"
done
python - "$OUT" <<'PY'
import json, sys
d = sys.argv[1]
a, b = (json.load(open(f"{d}/{k}.json")) for k in ("torch", "native"))
delta = abs(a["train_loss"] - b["train_loss"])
print(json.dumps({"torch_train_loss": a["train_loss"], "native_train_loss": b["train_loss"], "abs_delta": delta,
                  "threshold": 1e-2, "pass": delta <= 1e-2}))
sys.exit(0 if delta <= 1e-2 else 1)
PY
