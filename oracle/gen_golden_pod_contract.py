"""Generate tests/golden/controller_pod_contract.json: the literals the reference's RAG engine controller puts into the pod
spec (pkg/ragengine/manifests/manifests.go:116-134, 146-279; pkg/ragengine/controllers/preset_rag.go:33-64, 186) --
lifecycle hook script path and verbs, the environment variables it sets, the container command, port and probe path.
Run: python oracle/gen_golden_pod_contract.py <reference checkout>"""
import json
import os
import re
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "controller_pod_contract.json")


def main(ref_root):
    go = os.path.join(ref_root, "pkg", "ragengine")
    man = open(os.path.join(go, "manifests", "manifests.go")).read()
    pre = open(os.path.join(go, "controllers", "preset_rag.go")).read()
    hook_path = re.search(r'"(/app/ragengine/lifecycle/hooks\.py)"', man).group(1)
    verbs = [v for v in ("poststart", "prestop") if f"python3 {hook_path} {v}" in man or f'"{v}"' in man]
    env = [e for e in ("POD_NAME", "POD_UID", "DEFAULT_VECTOR_DB_PERSIST_DIR") if f'Name:  "{e}"' in man or f'Name: "{e}"' in man]
    command = re.search(r'utils\.ShellCmd\("([^"]+)"\)', pre).group(1)
    port = int(re.search(r"PortInferenceServer\s*=\s*(\d+)", pre).group(1))
    probe = re.search(r'ProbePath\s*=\s*"([^"]+)"', pre).group(1)
    out = {"meta": {"source": "pkg/ragengine/manifests/manifests.go, pkg/ragengine/controllers/preset_rag.go",
                    "generator": "oracle/gen_golden_pod_contract.py"},
           "hook_path": hook_path, "hook_verbs": verbs, "env": env, "command": command, "port": port, "probe_path": probe}
    json.dump(out, open(OUT, "w"), indent=1, sort_keys=True)
    print(out)


if __name__ == "__main__":
    main(sys.argv[1])
