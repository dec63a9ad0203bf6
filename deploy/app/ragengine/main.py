#!/usr/bin/env python3
"""Image entry shim. The unmodified KAITO controller starts the pod with
`/bin/sh -c "python3 main.py"` in WORKDIR /app/ragengine (pkg/ragengine/controllers/preset_rag.go:186,
docker/ragengine/service/Dockerfile:39), so the H100 image keeps a file of that name that hands over to the
CUDA-backed service (port 5000, GET /health for the probes: preset_rag.go:33-64)."""
import os
import sys

sys.path.insert(0, os.environ.get("KRAG_HOME", "/opt/kaito_b200"))
from kaito_b200.service import main  # noqa: E402

if __name__ == "__main__":
    main()
