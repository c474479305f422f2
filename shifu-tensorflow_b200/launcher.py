"""Node launcher: one YARN worker container -> one data-parallel rank per GPU of the node (SURVEY.md 8f rank 4).

The stock executor starts ONE python process per worker container (TensorflowTaskExecutor.java:300-317) and the
application master expects ONE metrics line per worker container and epoch (SocketServer.java:71-89,
TensorflowSession.java:515-549).  An H100 node has up to 8 GPUs, so this script is what
`shifu.application.python-script-path` points at when a container owns more than one GPU: it is started with the
executor's usual environment (the same contract `trainer.py` honours) and

  * starts G local ranks (`python -m shifu_tensorflow_b200.trainer`), G = $SB_LOCAL_GPUS or the number of sm_90
    devices, with the contract rewritten for a world of WORKER_CNT * G ranks:
        WORKER_CNT'   = WORKER_CNT * G          TASK_ID' = TASK_ID * G + g          LOCAL_RANK = SB_DEVICE = g
        CLUSTER_SPEC' = every worker address repeated G times (only worker[0], the NCCL-id rendezvous of global
                        rank 0, is ever dialled)
        SB_ROW_SHARD  = "g/G": the container's files are read by every local rank, rank g keeps rows g::G
        SOCKET_SERVER_PORT' = a relay socket owned by this launcher
  * relays metrics: per epoch it waits for the line of every local rank and sends ONE line to the executor's
    SOCKET_SERVER_PORT in the reference format, worker_index = this container's TASK_ID, time = max, losses = mean;
  * propagates exit codes: 0 only if every rank exits 0; the first failing rank's code otherwise, after the
    remaining ranks (exact PIDs) have been terminated - the chief's non-zero exit fails the job
    (TensorflowSession.java:437-452);
  * JOB_NAME=ps: idles exactly like `trainer.py` (there is no parameter server).
"""
from __future__ import annotations

import json
import logging
import os
import signal
import socket
import subprocess
import sys
import threading
import time
from typing import Dict, List, Optional, Sequence

LINE_KEYS = ("worker_index", "time", "current_epoch", "training_loss", "valid_loss")


def parse_metrics_line(line: str) -> Dict[str, float]:
    """"worker_index:0,time:1.5,current_epoch:3,training_loss:0.2,valid_loss:0.3" -> dict (SocketServer.java:71-89)"""
    out = {}
    for part in line.strip().split(","):
        k, v = part.split(":", 1)
        out[k] = float(v)
    missing = [k for k in LINE_KEYS if k not in out]
    if missing:
        raise ValueError("metrics line without %s: %r" % (missing, line))
    return out


def aggregate_lines(container_index: int, lines: Sequence[str]) -> str:
    """one line per local rank of the same epoch -> the container's line: time = max, losses = mean"""
    recs = [parse_metrics_line(l) for l in lines]
    epochs = {int(r["current_epoch"]) for r in recs}
    if len(epochs) != 1:
        raise ValueError("local ranks disagree on the epoch: %s" % sorted(epochs))
    n = float(len(recs))
    return "worker_index:{},time:{},current_epoch:{},training_loss:{},valid_loss:{}\n".format(
        str(container_index), str(max(r["time"] for r in recs)), str(epochs.pop()),
        str(sum(r["training_loss"] for r in recs) / n), str(sum(r["valid_loss"] for r in recs) / n))


def child_env(env: Dict[str, str], g: int, n_local: int, relay_port: int) -> Dict[str, str]:
    """the executor's environment rewritten for local rank g of n_local"""
    e = dict(env)
    workers = int(env["WORKER_CNT"])
    task = int(env["TASK_ID"])
    spec = json.loads(env["CLUSTER_SPEC"])
    spec["worker"] = [addr for addr in spec.get("worker", []) for _ in range(n_local)]
    e["WORKER_CNT"] = str(workers * n_local)
    e["TASK_ID"] = str(task * n_local + g)
    e["CLUSTER_SPEC"] = json.dumps(spec)
    e["LOCAL_RANK"] = str(g)
    e["SB_DEVICE"] = str(g)
    e["SB_ROW_SHARD"] = "%d/%d" % (g, n_local)
    e["SOCKET_SERVER_PORT"] = str(relay_port)
    return e


class MetricsRelay(threading.Thread):
    """Accepts the local ranks' metric connections, forwards one aggregated line per epoch upstream."""

    def __init__(self, container_index: int, n_local: int, upstream_port: Optional[int]):
        super().__init__(daemon=True)
        self.container_index, self.n_local, self.upstream_port = container_index, n_local, upstream_port
        self.srv = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
        self.srv.bind(("127.0.0.1", 0))
        self.srv.listen(n_local)
        self.port = self.srv.getsockname()[1]
        self.sent: List[str] = []            # what went upstream (also kept for tests)
        self._by_epoch: Dict[int, List[str]] = {}
        self._lock = threading.Lock()
        self._up: Optional[socket.socket] = None
        self._closing = False

    def _upstream(self) -> Optional[socket.socket]:
        if self._up is None and self.upstream_port is not None:
            self._up = socket.create_connection(("127.0.0.1", self.upstream_port), timeout=30)
        return self._up

    def _on_line(self, line: str):
        ep = int(parse_metrics_line(line)["current_epoch"])
        with self._lock:
            bucket = self._by_epoch.setdefault(ep, [])
            bucket.append(line)
            if len(bucket) < self.n_local:
                return
            del self._by_epoch[ep]
            out = aggregate_lines(self.container_index, bucket)
            self.sent.append(out)
            up = self._upstream()
            if up is not None:
                up.sendall(out.encode("utf8"))

    def _serve(self, conn: socket.socket):
        buf = b""
        with conn:
            while True:
                chunk = conn.recv(4096)
                if not chunk:
                    break
                buf += chunk
                while b"\n" in buf:
                    raw, buf = buf.split(b"\n", 1)
                    if raw.strip():
                        self._on_line(raw.decode("utf8"))

    def run(self):
        self.srv.settimeout(0.2)
        workers = []
        while not self._closing:
            try:
                conn, _ = self.srv.accept()
            except socket.timeout:
                continue
            except OSError:
                break
            th = threading.Thread(target=self._serve, args=(conn,), daemon=True)
            th.start()
            workers.append(th)
        for th in workers:
            th.join(timeout=5)

    def close(self):
        """stop accepting, let the per-connection readers drain what the ranks sent before they exited, then hang up"""
        self._closing = True
        if self.is_alive():
            self.join(timeout=10)
        try:
            self.srv.close()
        finally:
            if self._up is not None:
                self._up.close()


def local_gpu_count(env: Dict[str, str]) -> int:
    if env.get("SB_LOCAL_GPUS"):
        return max(1, int(env["SB_LOCAL_GPUS"]))
    from . import _capi as capi
    return max(1, capi.device_count())


def main(env: Optional[Dict[str, str]] = None, worker_cmd: Optional[Sequence[str]] = None) -> int:
    env = dict(os.environ if env is None else env)
    logging.basicConfig(level=logging.INFO, format='%(asctime)s %(name)-12s %(levelname)-8s %(message)s')
    if env["JOB_NAME"] == "ps":
        from . import trainer
        return trainer.main(env=env)
    n_local = local_gpu_count(env)
    container = int(env["TASK_ID"])
    upstream = int(env["SOCKET_SERVER_PORT"]) if env.get("SB_REQUIRE_SOCKET", "1") != "0" else None
    relay = MetricsRelay(container, n_local, upstream)
    relay.start()
    cmd = list(worker_cmd) if worker_cmd else [sys.executable, "-m", "shifu_tensorflow_b200.trainer"]
    procs = [subprocess.Popen(cmd, env=child_env(env, g, n_local, relay.port)) for g in range(n_local)]
    logging.info("container %d: started %d local ranks (pids %s)", container, n_local, [p.pid for p in procs])

    def forward(signum, _frame):            # the executor kills us -> take the ranks down too (exact PIDs only)
        for p in procs:
            if p.poll() is None:
                p.send_signal(signum)
    old = {s: signal.signal(s, forward) for s in (signal.SIGTERM, signal.SIGINT)} if threading.current_thread() is threading.main_thread() else {}

    rc = 0
    try:
        pending = set(range(n_local))
        while pending:
            for g in sorted(pending):
                code = procs[g].poll()
                if code is None:
                    continue
                pending.discard(g)
                if code != 0 and rc == 0:
                    rc = code if code > 0 else 128 - code      # killed by signal s -> 128 + s, like a shell reports it
                    logging.error("local rank %d exited with %d; stopping the other ranks", g, code)
                    for h in pending:
                        procs[h].terminate()
            time.sleep(0.05)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for s, h in old.items():
            signal.signal(s, h)
        relay.close()
    return rc


if __name__ == "__main__":
    sys.exit(main())
