"""com.nvidia.spark.rapids.jni.BloomFilter (BloomFilter.java:26-119) over the C ABI (include/srj_b200.h: srj_bloom_filter_*).

The device side of Spark's runtime bloom-filter join: BloomFilterAggregate builds a filter on the small side of a join
(`create`, `put`, then `merge` of the per-task partial filters) and BloomFilterMightContain probes the large side with it
(`probe`).  A filter is a LIST scalar whose one row is the UINT8 bytes of Spark's serialized V1 / V2 filter.

    f = BloomFilter.create(BloomFilter.VERSION_2, numHashes, bloomFilterBits, seed)   # Scalar
    BloomFilter.put(f, keys)                                                          # keys: INT64 ColumnView
    m = BloomFilter.merge(list_column([f, g]))                                        # LIST<UINT8> of F filters
    hits = BloomFilter.probe(m, keys)                                                 # BOOL8, the keys' null mask
    hits = BloomFilter.probe(serialized_bytes_tensor, keys)                           # probebuffer

Argument errors Java reports as IllegalArgumentException raise ValueError; errors of the native layer raise
CudfException, as the reference's JNI layer does.
"""
import ctypes as C
import warnings
from typing import Optional, Sequence

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _empty, _stream_ptr

INT32_MAX = 2**31 - 1


class Scalar:
    """ai.rapids.cudf.Scalar.  Of type LIST<UINT8> (dtype None): one row holding the bytes of one serialized filter.  Of a
    fixed-width type: `data` holds the value's bytes and `valid` one device byte, non-zero when the scalar is valid, as
    cudf::scalar holds them on the device (Arithmetic.multiply reads both there)."""

    def __init__(self, data: torch.Tensor, dtype: Optional[DType] = None, valid: Optional[torch.Tensor] = None):
        self.data = data
        self.dtype = dtype
        self.valid = valid

    _NUMPY = {DType.INT8: "int8", DType.INT16: "int16", DType.INT32: "int32", DType.INT64: "int64", DType.FLOAT32: "float32",
              DType.FLOAT64: "float64"}

    @staticmethod
    def _fixed(type_id: int, value, device=None) -> "Scalar":
        import numpy as np
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        raw = np.array([0 if value is None else value], dtype=Scalar._NUMPY[type_id]).view(np.uint8)
        return Scalar(torch.from_numpy(raw.copy()).to(dev), DType(type_id),
                      torch.tensor([value is not None], dtype=torch.uint8, device=dev))

    @staticmethod
    def fromByte(v, device=None) -> "Scalar":
        return Scalar._fixed(DType.INT8, v, device)

    @staticmethod
    def fromShort(v, device=None) -> "Scalar":
        return Scalar._fixed(DType.INT16, v, device)

    @staticmethod
    def fromInt(v, device=None) -> "Scalar":
        return Scalar._fixed(DType.INT32, v, device)

    @staticmethod
    def fromLong(v, device=None) -> "Scalar":
        return Scalar._fixed(DType.INT64, v, device)

    @staticmethod
    def fromFloat(v, device=None) -> "Scalar":
        return Scalar._fixed(DType.FLOAT32, v, device)

    @staticmethod
    def fromDouble(v, device=None) -> "Scalar":
        return Scalar._fixed(DType.FLOAT64, v, device)

    @staticmethod
    def fromString(v, device=None) -> "Scalar":
        """A STRING scalar: `data` holds its UTF-8 bytes (str) or the bytes given, on the device; None is a null scalar."""
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        raw = b"" if v is None else (v.encode() if isinstance(v, str) else bytes(v))
        return Scalar(torch.tensor(list(raw), dtype=torch.uint8, device=dev), DType(DType.STRING),
                      torch.tensor([v is not None], dtype=torch.uint8, device=dev))

    @staticmethod
    def fromNull(dtype: DType, device=None) -> "Scalar":
        return Scalar._fixed(dtype.type_id, None, device)

    def getType(self) -> DType:
        return DType(DType.LIST) if self.dtype is None else self.dtype

    def isValid(self) -> bool:
        return self.valid is None or bool(self.valid.item())

    def getListAsColumnView(self) -> ColumnView:
        return ColumnView(DType.UINT8, self.data.numel(), self.data, null_count=0)

    def close(self):
        self.data = self.valid = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def list_column(filters: Sequence[Scalar]) -> ColumnVector:
    """The LIST<UINT8> column of ColumnVector.concatenate(ColumnVector.fromScalar(f, 1), ...): one row per filter."""
    datas = [f.data for f in filters]
    dev = datas[0].device
    child = torch.cat(datas) if datas else _empty(0, torch.uint8, dev)
    lens = torch.tensor([0] + [d.numel() for d in datas], dtype=torch.int64)
    offsets = torch.cumsum(lens, 0).to(torch.int32).to(dev)
    return ColumnVector(DType.LIST, len(datas), None, None, offsets, ColumnVector(DType.UINT8, child.numel(), child),
                        null_count=0)


def _device_of(t: Optional[torch.Tensor]):
    return t.device if t is not None else torch.device("cuda", torch.cuda.current_device())


def _check_input(cv: ColumnView, what: str):
    if cv is None:
        raise TypeError(f"{what}: input column is null")                          # JNI_NULL_CHECK
    if cv.dtype.type_id != DType.INT64:
        raise N.CudfException(f"{what}: bloom filters take one INT64 column (type id {cv.dtype.type_id})")


class BloomFilter:
    VERSION_1 = 1
    VERSION_2 = 2
    DEFAULT_SEED = 0

    @staticmethod
    def create(*args) -> Scalar:
        """create(version, numHashes, bloomFilterBits, seed), or the deprecated create(numHashes, bloomFilterBits)
        (V1, DEFAULT_SEED).  The bit count is rounded up to a multiple of 64."""
        if len(args) == 2:
            warnings.warn("BloomFilter.create(numHashes, bloomFilterBits) is deprecated: use create(version, numHashes, "
                          "bloomFilterBits, seed)", DeprecationWarning, stacklevel=2)
            args = (BloomFilter.VERSION_1, args[0], args[1], BloomFilter.DEFAULT_SEED)
        version, num_hashes, bits, seed = (int(a) for a in args)
        if version not in (BloomFilter.VERSION_1, BloomFilter.VERSION_2):          # BloomFilter.java:64-72
            raise ValueError("Bloom filter version must be 1 or 2")
        if num_hashes <= 0:
            raise ValueError("Bloom filters must have a positive hash count")
        if bits <= 0:
            raise ValueError("Bloom filters must have a positive number of bits")
        if bits > INT32_MAX * 64:                                                  # BloomFilterJni.cpp:40-46
            raise ValueError("bloom filter bit count must be positive and less than or equal to the maximum supported size")
        seed = ((seed + 2**31) % 2**32) - 2**31                                    # a Java int
        lib = N.lib()
        longs, total = C.c_int32(0), C.c_int64(0)
        N.check(lib.srj_bloom_filter_sizes(version, num_hashes, bits, C.byref(longs), C.byref(total)), "BloomFilter.create")
        dev = torch.device("cuda", torch.cuda.current_device())
        buf = _empty(total.value, torch.uint8, dev)
        N.check(lib.srj_bloom_filter_init(version, num_hashes, longs.value, seed, buf.data_ptr(), _stream_ptr()),
                "BloomFilter.create")
        return Scalar(buf)

    @staticmethod
    def put(bloomFilter: Scalar, cv: ColumnView) -> None:
        """Set the bits of every non-null value of the INT64 column `cv`."""
        if bloomFilter is None or bloomFilter.data is None:
            raise TypeError("BloomFilter.put: bloom filter is null")
        _check_input(cv, "BloomFilter.put")
        buf = bloomFilter.data
        with torch.cuda.device(buf.device):
            N.check(N.lib().srj_bloom_filter_put(buf.data_ptr(), buf.numel(), C.byref(cv._c()), _stream_ptr()),
                    "BloomFilter.put")

    @staticmethod
    def merge(bloomFilters: ColumnView) -> Scalar:
        """OR of the filters in the rows of a LIST<UINT8> column; they must all share version, numHashes, seed and size."""
        if bloomFilters is None:
            raise TypeError("BloomFilter.merge: input column is null")
        if bloomFilters.dtype.type_id != DType.LIST or bloomFilters.child is None:
            raise N.CudfException("BloomFilter.merge: expected a LIST<UINT8> column of serialized filters")
        child = bloomFilters.child.data
        n = bloomFilters.size
        nbytes = child.numel() if child is not None else 0
        dev = _device_of(child if child is not None else bloomFilters.offsets)
        with torch.cuda.device(dev):
            lib = N.lib()
            out = _empty(nbytes // n if n > 0 else 0, torch.uint8, dev)
            ws = _empty(lib.srj_bloom_filter_merge_workspace_bytes(), torch.uint8, dev)
            N.check(lib.srj_bloom_filter_merge(child.data_ptr() if nbytes else None, nbytes, n,
                                               out.data_ptr() if out.numel() else None, ws.data_ptr(), _stream_ptr()),
                    "BloomFilter.merge")
            return Scalar(out)

    @staticmethod
    def probe(bloomFilter, cv: ColumnView) -> ColumnVector:
        """BOOL8 column: true where the value may be in the filter, false where it is not; nulls of `cv` stay null.
        `bloomFilter` is a Scalar (probe) or a device uint8 tensor holding a serialized filter (probebuffer)."""
        if bloomFilter is None:
            raise TypeError("BloomFilter.probe: bloom filter is null")
        buf = bloomFilter.data if isinstance(bloomFilter, Scalar) else bloomFilter
        if buf is None:
            raise TypeError("BloomFilter.probe: bloom filter is null")
        return BloomFilter._probe(buf.data_ptr(), buf.numel(), cv, buf.device)

    @staticmethod
    def probebuffer(address: int, length: int, cv: ColumnView) -> ColumnVector:
        """probe(BaseDeviceMemoryBuffer, cv) by address and length of the device buffer."""
        return BloomFilter._probe(int(address), int(length), cv, _device_of(cv.data))

    @staticmethod
    def _probe(address: int, length: int, cv: ColumnView, dev) -> ColumnVector:
        _check_input(cv, "BloomFilter.probe")
        n = cv.size
        with torch.cuda.device(dev):
            out = _empty(n, torch.uint8, dev)
            mask = _empty((n + 31) // 32, torch.int32, dev) if cv.mask is not None else None
            N.check(N.lib().srj_bloom_filter_probe(address or None, length, C.byref(cv._c()), out.data_ptr() if n else None,
                                                   mask.data_ptr() if mask is not None and n else None, _stream_ptr()),
                    "BloomFilter.probe")
            return ColumnVector(DType.BOOL8, n, out, mask, null_count=cv.getNullCount())
