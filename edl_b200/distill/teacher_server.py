"""A teacher inference server: serves a PyTorch module over gRPC (``edl.predict.PredictService``).

Replaces ``python -m paddle_serving_server_gpu.serve --model ... --port ... --gpu_ids ...``
(README.md:59-63, example/distill/resnet/scripts/start_local_teacher.sh:24-30).  Requests from many
students are micro-batched into one forward pass per GPU tick.

    python -m paddle_edl.distill.teacher_server --model resnext101_32x16d --port 9292 --gpu_ids 0
"""
import argparse
import logging
import queue
import threading
import time

import numpy as np
import torch

from ..protos import rpc, schema
from ..utils import exceptions

logger = logging.getLogger("edl.teacher")


class TeacherServer:
    def __init__(self, model, feed_names, fetch_names, feed_shapes=None, device="cpu", dtype=torch.float32,
                 port=0, host="0.0.0.0", max_batch=64, max_wait_ms=2.0, workers=8, postprocess=None):
        """``model(*feeds) -> tensor | tuple | dict``; outputs are matched to ``fetch_names`` in order."""
        self.model = model.to(device).eval() if isinstance(model, torch.nn.Module) else model
        self.feed_names, self.fetch_names = list(feed_names), list(fetch_names)
        self.feed_shapes = feed_shapes or {}
        self.device, self.dtype = torch.device(device), dtype
        self.port, self.host = port, host
        self.max_batch, self.max_wait = max_batch, max_wait_ms / 1000.0
        self.postprocess = postprocess
        self._q = queue.Queue()
        self._stop = threading.Event()
        self._server = None
        self._workers = workers
        self.served = 0

    # ------------------------------------------------------------------ rpc handlers
    def _get_conf(self, request, context):
        import json

        return schema.predict.ConfResponse(feed_names=self.feed_names, fetch_names=self.fetch_names,
                                           feed_shapes_json=json.dumps(self.feed_shapes))

    def _predict(self, request, context):
        res = schema.predict.PredictResponse()
        try:
            feeds = {t.name: np.frombuffer(t.data, dtype=np.dtype(t.dtype)).reshape(list(t.shape))
                     for t in request.feeds}
            slot = {"feeds": feeds, "done": threading.Event(), "out": None, "err": None}
            self._q.put(slot)
            slot["done"].wait()
            if slot["err"] is not None:
                raise slot["err"]
            want = list(request.fetch) or self.fetch_names
            for name in want:
                arr = np.ascontiguousarray(slot["out"][name])
                res.outputs.append(schema.predict.Tensor(name=name, dtype=str(arr.dtype), shape=list(arr.shape),
                                                         data=arr.tobytes()))
        except Exception as e:  # noqa: BLE001
            exceptions.serialize(res.status, e if isinstance(e, exceptions.EdlException)
                                 else exceptions.EdlInternalError(repr(e)))
        return res

    # ------------------------------------------------------------------ batching loop
    @torch.no_grad()
    def _run_batch(self, slots):
        sizes = [len(next(iter(s["feeds"].values()))) for s in slots]
        if hasattr(self.model, "forward_requests"):
            # the model collates itself (sequence teachers pack requests of different lengths)
            out = self.model.forward_requests([[s["feeds"][name] for name in self.feed_names] for s in slots])
        else:
            feeds = []
            for name in self.feed_names:
                arr = np.concatenate([s["feeds"][name] for s in slots], 0)
                t = torch.from_numpy(np.ascontiguousarray(arr)).to(self.device)
                if t.is_floating_point():
                    t = t.to(self.dtype)
                    if t.dim() == 4 and self.device.type == "cuda":
                        t = t.contiguous(memory_format=torch.channels_last)
                feeds.append(t)
            out = self.model(*feeds)
        if self.postprocess is not None:
            out = self.postprocess(out)
        if isinstance(out, dict):
            outs = {k: out[k] for k in self.fetch_names}
        else:
            if not isinstance(out, (tuple, list)):
                out = (out,)
            outs = dict(zip(self.fetch_names, out))
        outs = {k: v.float().cpu().numpy() for k, v in outs.items()}
        off = 0
        for s, n in zip(slots, sizes):
            s["out"] = {k: v[off:off + n] for k, v in outs.items()}
            off += n
            s["done"].set()
        self.served += sum(sizes)

    def _loop(self):
        while not self._stop.is_set():
            try:
                first = self._q.get(timeout=0.1)
            except queue.Empty:
                continue
            slots, n = [first], len(next(iter(first["feeds"].values())))
            deadline = time.time() + self.max_wait
            while n < self.max_batch:
                try:
                    s = self._q.get(timeout=max(0.0, deadline - time.time()))
                except queue.Empty:
                    break
                slots.append(s)
                n += len(next(iter(s["feeds"].values())))
            try:
                self._run_batch(slots)
            except Exception as e:  # noqa: BLE001
                logger.exception("teacher forward failed")
                for s in slots:
                    s["err"] = e
                    s["done"].set()

    # ------------------------------------------------------------------ lifecycle
    def start(self):
        self._server = rpc.make_server(self._workers)
        rpc.add_service(self._server, "edl.predict.PredictService",
                        {"Predict": self._predict, "GetConf": self._get_conf})
        self.port = self._server.add_insecure_port("{}:{}".format(self.host, self.port))
        assert self.port > 0, "cannot bind teacher server"
        self._server.start()
        self._t = threading.Thread(target=self._loop, daemon=True, name="teacher-batcher")
        self._t.start()
        logger.info("teacher serving %s -> %s on port %d", self.feed_names, self.fetch_names, self.port)
        return self

    @property
    def endpoint(self):
        return "127.0.0.1:%d" % self.port

    def stop(self):
        self._stop.set()
        if self._server is not None:
            self._server.stop(0)
            self._server = None

    def __enter__(self):
        return self.start()

    def __exit__(self, *exc):
        self.stop()


def build_model(name):
    from ..models import teacher_zoo

    return teacher_zoo.build(name)


def fp8_scaling(net, requested=None):
    """The ``--fp8`` scaling for teacher network ``net``.  ``requested`` None picks the model's default: ``block`` for a
    sequence teacher (one that serves ``forward_requests``), ``tensor`` for an image teacher.  A sequence teacher offers
    block scaling only: it raises ValueError for any other request."""
    sequence = hasattr(net, "forward_requests")
    if requested is None:
        return "block" if sequence else "tensor"
    if sequence and requested != "block":
        raise ValueError("--fp8_scaling %s is not available for a sequence teacher: use --fp8_scaling block "
                         "(the default for it)" % requested)
    return requested


def main(argv=None):
    ap = argparse.ArgumentParser(description="EDL teacher inference server")
    ap.add_argument("--model", required=True, help="teacher_zoo name, e.g. resnext101_32x16d / mnist_cnn / ernie_base")
    ap.add_argument("--weights", default=None,
                    help="state dict to load (.safetensors or a torch file); sequence teachers take the BERT layout. "
                         "Without it the weights are random")
    ap.add_argument("--port", type=int, default=9292)
    ap.add_argument("--gpu_ids", type=str, default="0")
    ap.add_argument("--thread", type=int, default=4)
    ap.add_argument("--max_batch", type=int, default=64)
    ap.add_argument("--mem_optim", action="store_true", help="accepted for CLI parity; no-op")
    ap.add_argument("--fp8", action="store_true",
                    help="e4m3 wgmma GEMMs for the 1x1 convolutions of an image teacher, or the encoder's linear layers "
                         "of a sequence teacher")
    ap.add_argument("--fp8_scaling", choices=("tensor", "block"), default=None,
                    help="with --fp8: 'tensor' = one activation scale per layer, calibrated on random data; 'block' = "
                         "per-row, per-128-channel activation scales computed as each layer runs (no calibration). "
                         "Default: 'tensor' for image teachers, 'block' (the only choice) for sequence teachers")
    args = ap.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    dev = "cuda:%s" % args.gpu_ids.split(",")[0] if torch.cuda.is_available() else "cpu"
    model, feed_names, fetch_names, feed_shapes = build_model(args.model)
    scaling = None
    if args.fp8:
        try:
            scaling = fp8_scaling(getattr(model, "net", model), args.fp8_scaling)
        except ValueError as e:
            ap.error(str(e))
    if args.weights:
        net = getattr(model, "net", model)
        if hasattr(net, "load_weights"):
            unused = net.load_weights(args.weights)
            logging.info("loaded %s (%d unused entries)", args.weights, len(unused))
        else:
            sd = torch.load(args.weights, map_location="cpu", weights_only=True)
            net.load_state_dict(sd.get("state_dict", sd))
    dtype = torch.bfloat16 if dev.startswith("cuda") else torch.float32
    srv = TeacherServer(model, feed_names, fetch_names, feed_shapes, device=dev, dtype=dtype, port=args.port,
                        max_batch=args.max_batch, workers=max(4, args.thread))
    net = getattr(srv.model, "net", srv.model)
    if args.fp8 and dev.startswith("cuda") and hasattr(net, "enable_fp8") and scaling == "block":
        logging.info("fp8 (block-scaled): converted %d layers", net.enable_fp8(scaling="block"))
    elif args.fp8 and dev.startswith("cuda") and hasattr(net, "enable_fp8"):
        shape = feed_shapes[feed_names[0]]
        calib = torch.randn(8, *shape, device=dev).to(dtype).contiguous(memory_format=torch.channels_last)
        logging.info("fp8: converted %d layers", net.enable_fp8(calib))
    srv.start()
    try:
        while True:
            time.sleep(3600)
    except KeyboardInterrupt:
        srv.stop()


if __name__ == "__main__":
    main()
