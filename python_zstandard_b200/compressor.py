"""ZstdCompressor -- the compression half of the reference API that sits on the batch path.

Mirrors c-ext/compressor.c: constructor :88-261 (same keyword arguments, defaults and error
texts), compress() :509-574 and multi_compress_to_buffer() :1341-1504.  The frames come from the
CUDA block compressor in libzb200 (zb_encode.cu); they are RFC 8878 zstd and decode with any zstd
decoder, but they are not byte-identical to CPU zstd's -- the parse is this project's own.
With dict_data, the last 32 KiB of the dictionary content act as match history in front of every frame, the frame
starts from the dictionary's repcodes, and its entropy tables are reused where that is cheaper ("repeat" FSE tables,
"treeless" literals), like the reference's ZSTD_compress_insertDictionary (zstd/zstd.c:28015-28180).
"""
import ctypes as C

import numpy as np

from . import _native
from .buffers import BufferWithSegments, BufferWithSegmentsCollection, DeviceBufferWithSegments
from .decompressor import _devices
from .dictionary import ZstdCompressionDict
from .errors import ZstdError

MAX_COMPRESSION_LEVEL = 22

# the reference's strategy numbers and knob bounds (c-ext/constants.c; zstd.h, 64-bit build)
STRATEGY_FAST, STRATEGY_DFAST, STRATEGY_GREEDY, STRATEGY_LAZY, STRATEGY_LAZY2 = 1, 2, 3, 4, 5
STRATEGY_BTLAZY2, STRATEGY_BTOPT, STRATEGY_BTULTRA, STRATEGY_BTULTRA2 = 6, 7, 8, 9
SEARCHLOG_MIN, SEARCHLOG_MAX = 1, 30
MINMATCH_MIN, MINMATCH_MAX = 3, 7
TARGETLENGTH_MIN, TARGETLENGTH_MAX = 0, 131072
_LAZY_STRATEGIES = (STRATEGY_GREEDY, STRATEGY_LAZY, STRATEGY_LAZY2)
_OUT_OF_BOUND = "unable to set compression context parameter: Parameter is out of bound"


class CParams(C.Structure):
    _fields_ = [("level", C.c_int32), ("write_checksum", C.c_uint32), ("write_content_size", C.c_uint32),
                ("dict_id", C.c_uint32), ("window_log", C.c_uint32), ("strategy", C.c_uint32), ("search_log", C.c_uint32),
                ("min_match", C.c_uint32)]


class ZstdCompressionParameters:
    """The subset of c-ext/compressionparams.c that reaches this backend: level, the three frame flags, window_log, and
    strategy = STRATEGY_GREEDY / STRATEGY_LAZY / STRATEGY_LAZY2 with search_log and min_match, which select the GPU's
    hash-chain lazy parse (2^min(search_log, 6) chain candidates per position, clamp(min_match, 4, 6)-byte hashes and
    matches; target_length is accepted and, as in the reference's lazy strategies, has no effect).  Values outside the
    reference's bounds raise its error.  Any other strategy, search_log / min_match / target_length without one of those
    three strategies, hash_log, chain_log and the LDM / job knobs configure CPU zstd's other strategies, which this backend
    does not have: anything but their defaults is rejected loudly."""

    _FIELDS = ("format", "compression_level", "window_log", "hash_log", "chain_log", "search_log", "min_match",
               "target_length", "strategy", "write_content_size", "write_checksum", "write_dict_id", "job_size",
               "overlap_log", "force_max_window", "enable_ldm", "ldm_hash_log", "ldm_min_match",
               "ldm_bucket_size_log", "ldm_hash_rate_log", "threads")

    def __init__(self, **kw):
        for k in kw:
            if k not in self._FIELDS:
                raise TypeError("'%s' is an invalid keyword argument" % k)
        self.format = kw.get("format", 0)
        self.compression_level = kw.get("compression_level", 0)
        self.write_content_size = kw.get("write_content_size", 1)
        self.write_checksum = kw.get("write_checksum", 0)
        self.write_dict_id = kw.get("write_dict_id", 0)
        self.threads = kw.get("threads", 0)
        wl = kw.get("window_log", 0) or 0
        if wl and not (10 <= wl <= 31):
            raise ValueError("window_log out of range")        # ZSTD_c_windowLog bounds, zstd/zstd.c:23003
        self.window_log = wl
        # ZSTD_CCtxParams_setParameter's bounds (zstd/zstd.c:23763-23783); 0 (and the binding's -1) mean "the level's"
        given = {k: kw.get(k) for k in ("search_log", "min_match", "target_length", "strategy") if kw.get(k) not in (0, -1, None)}
        bounds = {"search_log": (SEARCHLOG_MIN, SEARCHLOG_MAX), "min_match": (MINMATCH_MIN, MINMATCH_MAX),
                  "target_length": (TARGETLENGTH_MIN, TARGETLENGTH_MAX), "strategy": (STRATEGY_FAST, STRATEGY_BTULTRA2)}
        for k, v in given.items():
            if not bounds[k][0] <= v <= bounds[k][1]:
                raise ZstdError(_OUT_OF_BOUND)
        lazy = given.get("strategy") in _LAZY_STRATEGIES
        for k in ("hash_log", "chain_log", "search_log", "min_match", "target_length", "strategy",
                  "job_size", "overlap_log", "force_max_window", "enable_ldm", "ldm_hash_log", "ldm_min_match",
                  "ldm_bucket_size_log", "ldm_hash_rate_log"):
            if lazy and k in given:
                setattr(self, k, given[k])
                continue
            v = kw.get(k, 0)
            if v not in (0, -1, None):
                raise ZstdError("compression parameter %s is not supported by the GPU backend" % k)
            setattr(self, k, 0)
        # What the caller asked for, apart from the attributes: from_level fills the match-finder attributes in as reports
        # of the reference's choice for the level, and those never select the parse.
        self._lazy = given["strategy"] if lazy else 0

    # The level tables of the reference (zstd/zstd.c:30650-30756): four size classes (any / <= 256 KB / <= 128 KB / <= 16 KB),
    # row 0 = base of the negative levels, rows 1..22 = levels; columns: window_log, chain_log, hash_log, search_log, min_match,
    # target_length, strategy (1 fast .. 9 btultra2).  Data, restated; only window_log reaches this backend.
    _LEVEL_TABLES = (
        ((19, 12, 13, 1, 6, 1, 1), (19, 13, 14, 1, 7, 0, 1), (20, 15, 16, 1, 6, 0, 1), (21, 16, 17, 1, 5, 0, 2), (21, 18, 18, 1, 5, 0, 2), (21, 18, 19, 3, 5, 2, 3), (21, 18, 19, 3, 5, 4, 4), (21, 19, 20, 4, 5, 8, 4),
         (21, 19, 20, 4, 5, 16, 5), (22, 20, 21, 4, 5, 16, 5), (22, 21, 22, 5, 5, 16, 5), (22, 21, 22, 6, 5, 16, 5), (22, 22, 23, 6, 5, 32, 5), (22, 22, 22, 4, 5, 32, 6), (22, 22, 23, 5, 5, 32, 6), (22, 23, 23, 6, 5, 32, 6),
         (22, 22, 22, 5, 5, 48, 7), (23, 23, 22, 5, 4, 64, 7), (23, 23, 22, 6, 3, 64, 8), (23, 24, 22, 7, 3, 256, 9), (25, 25, 23, 7, 3, 256, 9), (26, 26, 24, 7, 3, 512, 9), (27, 27, 25, 9, 3, 999, 9)),
        ((18, 12, 13, 1, 5, 1, 1), (18, 13, 14, 1, 6, 0, 1), (18, 14, 14, 1, 5, 0, 2), (18, 16, 16, 1, 4, 0, 2), (18, 16, 17, 3, 5, 2, 3), (18, 17, 18, 5, 5, 2, 3), (18, 18, 19, 3, 5, 4, 4), (18, 18, 19, 4, 4, 4, 4),
         (18, 18, 19, 4, 4, 8, 5), (18, 18, 19, 5, 4, 8, 5), (18, 18, 19, 6, 4, 8, 5), (18, 18, 19, 5, 4, 12, 6), (18, 19, 19, 7, 4, 12, 6), (18, 18, 19, 4, 4, 16, 7), (18, 18, 19, 4, 3, 32, 7), (18, 18, 19, 6, 3, 128, 7),
         (18, 19, 19, 6, 3, 128, 8), (18, 19, 19, 8, 3, 256, 8), (18, 19, 19, 6, 3, 128, 9), (18, 19, 19, 8, 3, 256, 9), (18, 19, 19, 10, 3, 512, 9), (18, 19, 19, 12, 3, 512, 9), (18, 19, 19, 13, 3, 999, 9)),
        ((17, 12, 12, 1, 5, 1, 1), (17, 12, 13, 1, 6, 0, 1), (17, 13, 15, 1, 5, 0, 1), (17, 15, 16, 2, 5, 0, 2), (17, 17, 17, 2, 4, 0, 2), (17, 16, 17, 3, 4, 2, 3), (17, 16, 17, 3, 4, 4, 4), (17, 16, 17, 3, 4, 8, 5),
         (17, 16, 17, 4, 4, 8, 5), (17, 16, 17, 5, 4, 8, 5), (17, 16, 17, 6, 4, 8, 5), (17, 17, 17, 5, 4, 8, 6), (17, 18, 17, 7, 4, 12, 6), (17, 18, 17, 3, 4, 12, 7), (17, 18, 17, 4, 3, 32, 7), (17, 18, 17, 6, 3, 256, 7),
         (17, 18, 17, 6, 3, 128, 8), (17, 18, 17, 8, 3, 256, 8), (17, 18, 17, 10, 3, 512, 8), (17, 18, 17, 5, 3, 256, 9), (17, 18, 17, 7, 3, 512, 9), (17, 18, 17, 9, 3, 512, 9), (17, 18, 17, 11, 3, 999, 9)),
        ((14, 12, 13, 1, 5, 1, 1), (14, 14, 15, 1, 5, 0, 1), (14, 14, 15, 1, 4, 0, 1), (14, 14, 15, 2, 4, 0, 2), (14, 14, 14, 4, 4, 2, 3), (14, 14, 14, 3, 4, 4, 4), (14, 14, 14, 4, 4, 8, 5), (14, 14, 14, 6, 4, 8, 5),
         (14, 14, 14, 8, 4, 8, 5), (14, 15, 14, 5, 4, 8, 6), (14, 15, 14, 9, 4, 8, 6), (14, 15, 14, 3, 4, 12, 7), (14, 15, 14, 4, 3, 24, 7), (14, 15, 14, 5, 3, 32, 8), (14, 15, 15, 6, 3, 64, 8), (14, 15, 15, 7, 3, 256, 8),
         (14, 15, 15, 5, 3, 48, 9), (14, 15, 15, 6, 3, 128, 9), (14, 15, 15, 7, 3, 256, 9), (14, 15, 15, 8, 3, 256, 9), (14, 15, 15, 8, 3, 512, 9), (14, 15, 15, 9, 3, 512, 9), (14, 15, 15, 10, 3, 999, 9)),
    )

    @classmethod
    def _cparams_for(cls, level, source_size, dict_size):
        """ZSTD_getCParams(level, source_size, dict_size) restated: the row by size class (ZSTD_getCParamRowSize and
        ZSTD_getCParams_internal, zstd/zstd.c:30823-30871), then ZSTD_adjustCParams_internal in its "unknown" mode
        (:24427-24563: window downsized to the input, hash / chain logs to the window, the row-hash cap).  source_size 0 means
        unknown, as in c-ext/compressionparams.c:234-279."""
        unknown = source_size == 0
        if unknown:
            rsize = (1 << 64) - 1 if dict_size == 0 else dict_size + 499        # (UNKNOWN + dictSize + 500 wraps in the reference)
        else:
            rsize = source_size + dict_size
        table = (rsize <= 256 << 10) + (rsize <= 128 << 10) + (rsize <= 16 << 10)
        row = 3 if level == 0 else (0 if level < 0 else min(level, 22))
        wlog, clog, hlog, slog, mml, tlen, strat = cls._LEVEL_TABLES[table][row]
        if level < 0:
            tlen = -max(level, -(1 << 17))                                      # acceleration: ZSTD_minCLevel() = -ZSTD_TARGETLENGTH_MAX
        if not unknown and source_size <= (1 << 30) and dict_size <= (1 << 30):
            tsize = (source_size + dict_size) & 0xFFFFFFFF
            wlog = min(wlog, 6 if tsize < 64 else (tsize - 1).bit_length())
        if not unknown:
            # ZSTD_dictAndWindowLog: a window log that also reaches the dictionary
            dw = wlog
            if dict_size:
                wsize = 1 << wlog
                if wsize < dict_size + source_size:
                    dw = 31 if dict_size + wsize >= (1 << 31) else (dict_size + wsize - 1).bit_length()
            hlog = min(hlog, dw + 1)
            cycle = clog - (1 if strat >= 6 else 0)                            # ZSTD_cycleLog: binary-tree strategies count double
            if cycle > dw:
                clog -= cycle - dw
        wlog = max(wlog, 10)                                                    # ZSTD_WINDOWLOG_ABSOLUTEMIN
        if 3 <= strat <= 5:                                                     # the row-based match finder hashes at most 32 bits
            hlog = min(hlog, 24 + min(max(slog, 4), 6))
        return {"window_log": wlog, "chain_log": clog, "hash_log": hlog, "search_log": slog, "min_match": mml,
                "target_length": tlen, "strategy": strat}

    @classmethod
    def from_level(cls, level, source_size=0, dict_size=0, **kwargs):
        """ZstdCompressionParameters.from_level (c-ext/compressionparams.c:234-380): the parameters ZSTD_getCParams picks for
        (level, source_size, dict_size), each unless given.  window_log is the one that reaches this backend (frame header,
        block size); the match-finder columns are reported as attributes, like the reference's, and describe CPU strategies
        this backend replaces by its own parse of that level's class.  An explicit strategy=STRATEGY_GREEDY / _LAZY / _LAZY2
        keyword selects the GPU's lazy parse, with the search_log and min_match given or else reported for the level; other
        match-finder keywords are refused as by the constructor."""
        derived = cls._cparams_for(level, source_size, dict_size)
        if kwargs.get("window_log") in (None, 0, -1):
            kwargs["window_log"] = derived["window_log"]
        self = cls(compression_level=level, **kwargs)
        for k, v in derived.items():
            if k != "window_log" and kwargs.get(k) in (None, 0, -1):
                setattr(self, k, v)
        return self


class ZstdCompressor:
    def __init__(self, level=3, dict_data=None, compression_params=None, write_checksum=None,
                 write_content_size=None, write_dict_id=None, threads=0):
        if level > MAX_COMPRESSION_LEVEL:
            raise ValueError("level must be less than %d" % (MAX_COMPRESSION_LEVEL + 1))
        if dict_data is not None and not isinstance(dict_data, ZstdCompressionDict):
            raise TypeError("dict_data must be zstd.ZstdCompressionDict")
        if compression_params is not None and not isinstance(compression_params, ZstdCompressionParameters):
            raise TypeError("compression_params must be zstd.ZstdCompressionParameters")
        if compression_params is not None:
            if write_checksum is not None:
                raise ValueError("cannot define compression_params and write_checksum")
            if write_content_size is not None:
                raise ValueError("cannot define compression_params and write_content_size")
            if write_dict_id is not None:
                raise ValueError("cannot define compression_params and write_dict_id")
            if threads:
                raise ValueError("cannot define compression_params and threads")
            self._level = compression_params.compression_level or 3
            self._checksum = bool(compression_params.write_checksum)
            self._content_size = bool(compression_params.write_content_size)
            self._write_dict_id = bool(compression_params.write_dict_id)
            self._window_log = compression_params.window_log
            # an explicit greedy / lazy / lazy2 strategy; search_log and min_match 0 take level 3's (1 and 5, zb200.h)
            lz = compression_params._lazy
            self._lazy = (lz, compression_params.search_log if lz else 0, compression_params.min_match if lz else 0)
        else:
            self._window_log = 0
            self._lazy = (0, 0, 0)
            self._level = level
            # defaults: content size on, checksum off, dict id on (c-ext/compressor.c:213-227)
            self._checksum = bool(write_checksum) if write_checksum is not None else False
            self._content_size = bool(write_content_size) if write_content_size is not None else True
            self._write_dict_id = bool(write_dict_id) if write_dict_id is not None else True
        self._dict_data = dict_data
        self._threads = threads

    def _params(self):
        did = self._dict_data.dict_id() if (self._dict_data is not None and self._write_dict_id) else 0
        return CParams(self._level, int(self._checksum), int(self._content_size), did, self._window_log, *self._lazy)

    def _dict(self, ctx):
        return self._dict_data._ddict(ctx) if self._dict_data is not None else None

    def memory_size(self):
        return 0

    def frame_progression(self):
        return (0, 0, 0)

    # ------------------------------------------------------------------ one-shot
    def compress(self, data):
        view = memoryview(data)
        buf = np.frombuffer(view, dtype=np.uint8) if view.nbytes else np.zeros(0, dtype=np.uint8)
        ctx = _native.Context.get(_native.default_device())
        L = ctx.L
        seg = np.array([[0, len(buf)]], dtype=np.uint64)
        res = C.c_void_p()
        p = self._params()
        dd = self._dict(ctx)            # (takes ctx.lock itself when it has to build the digest)
        with ctx.lock:
            rc = L.zb200_compress_batch(ctx.h, buf.ctypes.data if len(buf) else None, seg.ctypes.data, 1, C.byref(p),
                                        dd, 0, C.byref(res))
        ctx.check(rc, "zb200_compress_batch")
        try:
            n = L.zb200_result_size(res)
            return C.string_at(L.zb200_result_data(res), n)
        finally:
            L.zb200_result_free(res)

    # ------------------------------------------------------------------ batch
    def multi_compress_to_buffer(self, data, threads=0):
        if isinstance(data, DeviceBufferWithSegments):
            return self._run_device(data)
        if isinstance(data, BufferWithSegments):
            sources = [data]
        elif isinstance(data, BufferWithSegmentsCollection):
            sources = data._buffers
        elif isinstance(data, list):
            sources = None
        else:
            raise TypeError("argument must be list of BufferWithSegments")
        L = _native.lib()
        results = []
        if sources is not None:
            count = sum(len(b) for b in sources)
            total = 0
            for b in sources:
                segs = np.frombuffer(b._segments, dtype=np.uint64).reshape(-1, 2)
                total += int(segs[:, 1].sum()) if len(segs) else 0
            if count == 0:
                raise ValueError("no source elements found")
            if total == 0:
                raise ValueError("source elements are empty")
            for b in sources:
                if len(b) == 0:
                    continue
                segs = np.frombuffer(b._segments, dtype=np.uint64).reshape(-1, 2)
                dat = np.frombuffer(b._data, dtype=np.uint8) if b.size else np.zeros(1, dtype=np.uint8)
                results.extend(self._run(dat.ctypes.data, segs, threads, keep=(dat,)))
            return BufferWithSegmentsCollection(*results)
        views = []
        for i, item in enumerate(data):
            try:
                v = memoryview(item)
            except TypeError:
                raise TypeError("item %d not a bytes like object" % i)
            if not v.contiguous:
                raise TypeError("item %d not a bytes like object" % i)
            views.append(v)
        if not views:
            raise ValueError("no source elements found")
        if sum(v.nbytes for v in views) == 0:
            raise ValueError("source elements are empty")
        lengths = np.array([v.nbytes for v in views], dtype=np.uint64)
        from .decompressor import ZstdDecompressor
        devs = _devices(threads)
        parts = ZstdDecompressor._split(None, lengths, len(devs))
        p = self._params()
        for di, (lo, hi) in enumerate(parts):
            ctx = _native.Context.get(devs[di])
            k = hi - lo
            arrs = [np.frombuffer(v, dtype=np.uint8) if v.nbytes else np.zeros(0, dtype=np.uint8) for v in views[lo:hi]]
            ptrs = (C.c_void_p * k)(*[a.ctypes.data if len(a) else None for a in arrs])
            lens = (C.c_size_t * k)(*[len(a) for a in arrs])
            res = C.c_void_p()
            dd = self._dict(ctx)
            with ctx.lock:
                rc = L.zb200_compress_batch_ptrs(ctx.h, ptrs, lens, k, C.byref(p), dd, 0, C.byref(res))
            ctx.check(rc, "zb200_compress_batch_ptrs")
            results.append(BufferWithSegments._from_result(ctx, res))
        return BufferWithSegmentsCollection(*results)

    def _run_device(self, data):
        """Device-resident segments -> device-resident frames (SURVEY.md section 8(f)-2)."""
        n = len(data)
        if n == 0:
            raise ValueError("no source elements found")
        segs = np.frombuffer(data._segments, dtype=np.uint64).reshape(-1, 2)
        if int(segs[:, 1].sum()) == 0:
            raise ValueError("source elements are empty")
        ctx = _native.Context.get(data.device)
        L = ctx.L
        dd = self._dict(ctx)
        p = self._params()
        res = C.c_void_p()
        with ctx.lock:
            rc = L.zb200_compress_batch(ctx.h, data._ptr, data._segments, n, C.byref(p), dd,
                                        _native.SRC_DEVICE | _native.DST_DEVICE | _native.SEGS_HOST, C.byref(res))
        ctx.check(rc, "zb200_compress_batch")
        return DeviceBufferWithSegments._from_result(ctx, res)

    # one call keeps the whole device busy for milliseconds per 128 KiB block, so sub-batches only pay once a
    # call is large enough that its upload is worth hiding (measured: 256 MiB in one piece 20.5 ms, in 4 pieces 29 ms)
    PIPELINE_DEPTH = 2
    SUB_BATCH_INPUT_BYTES = 1 << 30

    def _run(self, base_ptr, segs, threads, keep=()):
        """Device partition as in the reference (contiguous ranges by bytes), then sub-batches of each range
        kept in flight on extra contexts so that uploads, kernels and downloads overlap."""
        from .decompressor import ZstdDecompressor, _executor
        L = _native.lib()
        devs = _devices(threads)
        lens = np.ascontiguousarray(segs[:, 1])
        parts = ZstdDecompressor._split(None, lens, len(devs))
        p = self._params()
        jobs = []
        for di, (lo, hi) in enumerate(parts):
            nbytes = int(lens[lo:hi].sum())
            k = max(1, min((hi - lo) // 64 or 1, nbytes // self.SUB_BATCH_INPUT_BYTES))
            if k < 2:
                jobs.append((devs[di], 0, lo, hi))
                continue
            for i, (a, c) in enumerate(ZstdDecompressor._split(None, lens[lo:hi], k)):
                jobs.append((devs[di], i % self.PIPELINE_DEPTH, lo + a, lo + c))

        def run(job):
            dev, slot, lo, hi = job
            ctx = _native.Context.get(dev, slot)
            sub = np.ascontiguousarray(segs[lo:hi])
            return BufferWithSegments._from_result(ctx, self._launch(ctx, base_ptr, sub, hi - lo, p))

        if len(jobs) == 1:
            return [run(jobs[0])]
        return list(_executor(self.PIPELINE_DEPTH * len(parts)).map(run, jobs))

    def _launch(self, ctx, base_ptr, sub, n, p):
        res = C.c_void_p()
        dd = self._dict(ctx)
        with ctx.lock:
            rc = ctx.L.zb200_compress_batch(ctx.h, base_ptr, sub.ctypes.data, n, C.byref(p), dd, 0, C.byref(res))
        ctx.check(rc, "zb200_compress_batch")
        return res

    # ------------------------------------------------------------------ content-dictionary chains
    _FAR_WINDOW = (1 << 31) - (1 << 27)          # ZB_FAR_WINDOW (csrc/zb_common.cuh)

    def compress_content_dict_chain(self, chunks):
        """The inverse of ZstdDecompressor.decompress_content_dict_chain (not a method of the reference): frame k is chunks[k]
        compressed with chunks[k - 1] as a raw-content prefix, so that the decompressor rebuilds chunks[k] from frames[:k + 1].

        Frame 0 is what compress(chunks[0]) writes, with this compressor's dictionary, level, dictionary-ID flag and
        parameters -- except that the chain format needs content sizes, so every frame carries one whatever
        write_content_size says.  Frames 1.. are single-segment frames (the window is the content size) with no dictionary
        ID and a checksum when write_checksum is set; their match sources may lie anywhere in the previous chunk, where the
        reference's loop over ZSTD_CCtx_refPrefix reaches only its window.  The whole chain is one batch on the default
        device.  A chunk of 2 GiB - 128 MiB or more, or with its predecessor that many bytes, raises ZstdError: the chain
        decoder does not take it."""
        if not isinstance(chunks, list):
            raise TypeError("compress_content_dict_chain() argument 1 must be list, not %s" % type(chunks).__name__)
        if not chunks:
            raise ValueError("empty input chain")
        views = []
        for i, item in enumerate(chunks):
            try:
                v = memoryview(item)
            except TypeError:
                raise TypeError("item %d not a bytes like object" % i)
            if not v.contiguous:
                raise TypeError("item %d not a bytes like object" % i)
            views.append(v)
        for k, v in enumerate(views):
            if v.nbytes >= self._FAR_WINDOW or (k and views[k - 1].nbytes + v.nbytes >= self._FAR_WINDOW):
                raise ZstdError("chunk %d is too large for a content-dictionary chain: size, or previous plus own size, of "
                                "2 GiB - 128 MiB or more" % k)
        n = len(views)
        arrs = [np.frombuffer(v, dtype=np.uint8) if v.nbytes else np.zeros(0, dtype=np.uint8) for v in views]
        ctx = _native.Context.get(_native.default_device())
        L = ctx.L
        ptrs = (C.c_void_p * n)(*[a.ctypes.data if len(a) else None for a in arrs])
        lens = (C.c_size_t * n)(*[len(a) for a in arrs])
        p = self._params()
        p.write_content_size = 1
        dd = self._dict(ctx)
        res = C.c_void_p()
        with ctx.lock:
            rc = L.zb200_compress_chain(ctx.h, ptrs, lens, n, C.byref(p), dd, C.byref(res))
        ctx.check(rc, "zb200_compress_chain")
        try:
            base = L.zb200_result_data(res)
            segs = (_native.Segment * n).from_address(L.zb200_result_segments(res))
            return [_native.bytes_from_address(base + s.offset, s.length) for s in segs]
        finally:
            L.zb200_result_free(res)

    # ------------------------------------------------------------------ out of scope (SURVEY.md section 2, row 15)
    def _unsupported(self, *a, **k):
        raise NotImplementedError("streaming compression objects are outside the GPU batch path")

    stream_reader = stream_writer = read_to_iter = copy_stream = chunker = _unsupported

    def compressobj(self, size=-1):
        """c-ext/compressor.c:576-640; the frame is written in one piece at flush() (streams.py)."""
        from .streams import ZstdCompressionObj
        return ZstdCompressionObj(self, size)
