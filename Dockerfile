# CUDA 12.9 devel image + PyTorch; builds the sm_90a extension in-tree at image build time.
FROM nvcr.io/nvidia/pytorch:25.06-py3
WORKDIR /app
COPY . /app
RUN pip install --no-cache-dir click rich websockets psutil fastapi "uvicorn[standard]" pydantic loguru python-dotenv httpx requests safetensors \
 && python -c "import __graft_entry__ as g; g.build()"
ENV BEE2BEE_OFFLINE=1
EXPOSE 4001 8000
CMD ["python", "-m", "bee2bee_b200", "serve-hf", "--random-weights", "--model", "distilgpt2", "--api-port", "8000"]
