#!/usr/bin/env bash
# Provider launcher (parity: /root/reference/run.sh): builds the sm_90a extension if needed, then
# serves MODEL through PROVIDER (hf | ollama | hf_remote) with PIECES layer pieces.
set -euo pipefail
MODEL="${MODEL:-distilgpt2}"; PROVIDER="${PROVIDER:-hf}"; PORT="${PORT:-0}"; API_PORT="${API_PORT:-8000}"; PIECES="${PIECES:-1}"
python -c "import __graft_entry__ as g; g.build()" >/dev/null
exec python -m bee2bee_b200.p2p_runtime --register --model "$MODEL" --provider "$PROVIDER" --port "$PORT" \
     --api-port "$API_PORT" --pieces "$PIECES" ${BOOTSTRAP:+--bootstrap "$BOOTSTRAP"} ${ENDPOINT:+--endpoint "$ENDPOINT"}
