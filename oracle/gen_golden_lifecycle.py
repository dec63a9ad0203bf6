"""Generate tests/golden/lifecycle_reference.json: what the reference's PreStop / PostStart handlers
(presets/ragengine/lifecycle/manager.py, executed unmodified) do against a RAG service -- the HTTP requests they send, the
snapshot they write (directory name, metadata.json, the LATEST link) and the snapshot fields they read back.  The handlers
run against a recording stand-in for the service that answers every request with 200.  Volatile parts are replaced by
placeholders: <snap> = absolute snapshot directory, <ts> = its timestamp, <iso> = the metadata timestamp.
Run: python oracle/gen_golden_lifecycle.py <reference checkout>"""
import http.server
import importlib.util
import json
import os
import sys
import tempfile
import threading
import types

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "lifecycle_reference.json")
INDEXES = ["idx_a", "idx b"]                  # the second name needs URL quoting
POD_UID, POD_NAME = "0123456789abcdef", "ragengine-0"


def main(ref_root):
    requests_seen = []

    class Recorder(http.server.BaseHTTPRequestHandler):
        def _answer(self, body):
            requests_seen.append([self.command, self.path])
            data = json.dumps(body).encode()
            self.send_response(200)
            self.send_header("Content-Type", "application/json")
            self.send_header("Content-Length", str(len(data)))
            self.end_headers()
            self.wfile.write(data)

        def do_GET(self):
            self._answer(INDEXES if self.path == "/indexes" else {})

        def do_POST(self):
            self._answer({"message": "ok"})

        def log_message(self, *a):
            pass

    srv = http.server.ThreadingHTTPServer(("127.0.0.1", 0), Recorder)
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    url = f"http://127.0.0.1:{srv.server_address[1]}"

    spec = importlib.util.spec_from_file_location("ref_lifecycle_manager",
                                                  os.path.join(ref_root, "presets", "ragengine", "lifecycle", "manager.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    ref.wait_for_service.__defaults__ = (url + "/indexes", 60)
    for fn in (ref.get_indexes, ref.load_index, ref.persist_index):
        fn.__defaults__ = (url,)
    ref.time = types.SimpleNamespace(sleep=lambda s: None, time=ref.time.time)     # its 0.5 s rate limiting
    os.environ.update(POD_UID=POD_UID, POD_NAME=POD_NAME)

    base = tempfile.mkdtemp()
    assert ref.prestop_handler(base) == 0
    snaps = os.listdir(os.path.join(base, "systemsnapshots"))
    assert len(snaps) == 1
    snap_name = snaps[0]
    snap = os.path.join(base, "systemsnapshots", snap_name)
    ts = snap_name.split("_pod-")[0]

    def norm(s):
        return s.replace(snap, "<snap>").replace(ts, "<ts>")

    meta = json.load(open(os.path.join(snap, "metadata.json")))
    prestop = {"requests": [[m, norm(p)] for m, p in requests_seen],
               "snapshot_dir": norm(os.path.relpath(snap, base)),
               "snapshot_entries": sorted(os.listdir(snap)),
               "latest_link": norm(os.readlink(os.path.join(base, "LATEST"))),
               "metadata": {k: ("<iso>" if k == "timestamp" else v) for k, v in meta.items()}}

    requests_seen.clear()
    assert ref.poststart_handler(base) == 0
    poststart = {"requests": [[m, norm(p)] for m, p in requests_seen]}
    requests_seen.clear()
    os.remove(os.path.join(base, "LATEST"))          # LATEST lost: the newest snapshot directory is used and linked again
    assert ref.poststart_handler(base) == 0
    poststart_without_latest = {"requests": [[m, norm(p)] for m, p in requests_seen],
                                "latest_link": norm(os.readlink(os.path.join(base, "LATEST")))}
    srv.shutdown()

    out = {"meta": {"source": "presets/ragengine/lifecycle/manager.py executed unmodified against a recording service",
                    "generator": "oracle/gen_golden_lifecycle.py"},
           "env": {"POD_UID": POD_UID, "POD_NAME": POD_NAME}, "indexes": INDEXES,
           "prestop": prestop, "poststart": poststart, "poststart_without_latest": poststart_without_latest}
    json.dump(out, open(OUT, "w"), indent=1, sort_keys=True)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main(sys.argv[1])
