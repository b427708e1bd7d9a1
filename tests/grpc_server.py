"""tests only: a loopback gRPC server over grpc_transport.process_connections, and grpcio client helpers"""
import selectors
import socket
import threading
import time

from throttlecrab_b200 import grpc_transport as gt


class Server:
    """serves every accepted connection with process_connections(conns, limiter, now, ring) on one thread; `capture`
    keeps each connection's received bytes"""

    def __init__(self, limiter, ring=None, now_ns=None):
        self.limiter, self.ring, self.now_ns = limiter, ring, now_ns
        self.sock = socket.socket()
        self.sock.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        self.sock.bind(("127.0.0.1", 0))
        self.sock.listen(16)
        self.port = self.sock.getsockname()[1]
        self.capture = []
        self.stop = threading.Event()
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def _run(self):
        sel = selectors.DefaultSelector()
        self.sock.setblocking(False)
        sel.register(self.sock, selectors.EVENT_READ)
        conns = {}
        while not self.stop.is_set():
            ready = []
            for key, _ in sel.select(0.02):
                if key.fileobj is self.sock:
                    s, _ = self.sock.accept()
                    s.setblocking(False)
                    cn = gt.Connection()
                    cn.sock, cn.raw = s, bytearray()
                    self.capture.append(cn.raw)
                    conns[s] = cn
                    sel.register(s, selectors.EVENT_READ)
                    continue
                cn = conns[key.fileobj]
                try:
                    data = key.fileobj.recv(65536 - len(cn.buf))
                except (BlockingIOError, ConnectionError):
                    continue
                if not data:
                    sel.unregister(key.fileobj)
                    key.fileobj.close()
                    del conns[key.fileobj]
                    continue
                cn.buf += data
                cn.raw += data
                ready.append(cn)
            if ready:
                now = self.now_ns() if self.now_ns else time.time_ns()
                gt.process_connections(ready, self.limiter, now, self.ring)
                for cn in ready:
                    if cn.out:
                        cn.sock.setblocking(True)
                        cn.sock.sendall(bytes(cn.out))
                        cn.sock.setblocking(False)
                        cn.out.clear()
        for s in list(conns):
            s.close()
        sel.close()
        self.sock.close()

    def close(self):
        self.stop.set()
        self.thread.join(10)
        assert not self.thread.is_alive()


def request_bytes(key, max_burst, count, period, quantity):
    """ThrottleRequest as protobuf encodes it (zero fields omitted)"""
    def varint(v):
        v &= (1 << 64) - 1
        out = bytearray()
        while v >= 0x80:
            out.append(v & 0x7f | 0x80)
            v >>= 7
        out.append(v)
        return bytes(out)
    kb = key.encode() if isinstance(key, str) else key
    out = b"\x0a" + varint(len(kb)) + kb if kb else b""
    for tag, v in ((2, max_burst), (3, count), (4, period), (5, quantity)):
        if v:
            out += bytes([tag << 3]) + varint(v)
    return out


def throttle_stub(channel):
    return channel.unary_unary(gt.PATH.decode(), request_serializer=lambda b: b, response_deserializer=lambda b: b)
