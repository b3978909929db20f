"""An independent restatement of DISTINCTCOUNTHLL (DESIGN.md section 3.17) with Java's int / long semantics: stream-lib's
MurmurHash.hash(Object) and HyperLogLog (offerHashed, cardinality) as Pinot's DistinctCountHLLAggregationFunction uses
them.  Written from the rules, not from the library: the tests hold the device, the probe of pb200_hll.h and
query.hll_final to it."""
import math
import struct


def _int(x):
    """Java int of x (two's complement, 32 bits)."""
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >> 31 else x


def _ushr(x, n):
    """Java's >>> on an int."""
    return (x & 0xFFFFFFFF) >> n


def _imul(a, b):
    return _int(a * b)


M, R = _int(0x5BD1E995), 24


def hash_long(data):
    """MurmurHash.hashLong(long)."""
    data &= 0xFFFFFFFFFFFFFFFF
    data = data - (1 << 64) if data >> 63 else data
    h = 0
    k = _imul(_int(data), M)
    k ^= _ushr(k, R)
    k = _int(k)
    h ^= _imul(k, M)
    k = _imul(_int(data >> 32), M)
    k ^= _ushr(k, R)
    k = _int(k)
    h = _imul(h, M)
    h ^= _imul(k, M)
    h = _int(h)
    h ^= _ushr(h, 13)
    h = _imul(_int(h), M)
    h ^= _ushr(h, 15)
    return _int(h)


def hash_bytes(data, seed=-1):
    """MurmurHash.hash(byte[] data, int length, int seed); bytes are Java bytes (signed)."""
    length = len(data)
    sb = [b - 256 if b > 127 else b for b in data]
    h = _int(seed ^ length)
    len_4 = length >> 2
    for i in range(len_4):
        i4 = i << 2
        k = sb[i4 + 3]
        k = _int(k << 8)
        k = _int(k | (sb[i4 + 2] & 0xFF))
        k = _int(k << 8)
        k = _int(k | (sb[i4 + 1] & 0xFF))
        k = _int(k << 8)
        k = _int(k | (sb[i4 + 0] & 0xFF))
        k = _imul(k, M)
        k = _int(k ^ _ushr(k, R))
        k = _imul(k, M)
        h = _imul(h, M)
        h = _int(h ^ k)
    len_m = len_4 << 2
    left = length - len_m
    if left != 0:
        if left >= 3:
            h = _int(h ^ (sb[length - 3] << 16))
        if left >= 2:
            h = _int(h ^ (sb[length - 2] << 8))
        if left >= 1:
            h = _int(h ^ sb[length - 1])
        h = _imul(h, M)
    h = _int(h ^ _ushr(h, 13))
    h = _imul(h, M)
    h = _int(h ^ _ushr(h, 15))
    return h


def hash_value(v, data_type):
    """MurmurHash.hash(Object) of a value of the given stored type ("INT", "LONG", "FLOAT", "DOUBLE", "STRING")."""
    if data_type in ("INT", "LONG"):
        return hash_long(int(v))
    if data_type == "FLOAT":
        return hash_long(struct.unpack("<i", struct.pack("<f", float(v)))[0])
    if data_type == "DOUBLE":
        return hash_long(struct.unpack("<q", struct.pack("<d", float(v)))[0])
    return hash_bytes(v.encode("utf-8") if isinstance(v, str) else bytes(v))


def _nlz(x):
    x &= 0xFFFFFFFF
    return 32 - x.bit_length()


def registers(hashes, log2m):
    """HyperLogLog.offerHashed(int) of every hash: j = x >>> (32 - p), r = nlz((x << p) | (1 << (p - 1)) + 1) + 1."""
    reg = [0] * (1 << log2m)
    for x in hashes:
        j = _ushr(x, 32 - log2m)
        r = _nlz(_int(x << log2m) | ((1 << (log2m - 1)) + 1)) + 1
        if r > reg[j]:
            reg[j] = r
    return reg


def java_round(x):
    """Math.round(double) for x >= 0 or +inf: floor(x + 1/2) exactly, Long.MAX_VALUE at and beyond 2^63."""
    if x >= 2.0 ** 63:
        return (1 << 63) - 1
    f = math.floor(x)
    return int(f) + (1 if x - f >= 0.5 else 0)


def alpha_mm(p, m):
    if p == 4:
        return 0.673 * m * m
    if p == 5:
        return 0.697 * m * m
    if p == 6:
        return 0.709 * m * m
    return (0.7213 / (1 + 1.079 / m)) * m * m


def cardinality(reg, log2m):
    """HyperLogLog.cardinality(): registerSum accumulated in double in register order (exact here), then the estimate."""
    m = 1 << log2m
    register_sum = 0.0
    zeros = 0.0
    for v in reg:
        register_sum += 1.0 / (1 << v)
        if v == 0:
            zeros += 1
    estimate = alpha_mm(log2m, m) * (1 / register_sum)
    if estimate <= (5.0 / 2.0) * m:
        lc = m * math.log(m / zeros) if zeros else math.inf
        return java_round(lc)
    return java_round(estimate)


def hll(values, log2m=8, data_type="INT"):
    """DISTINCTCOUNTHLL of the distinct values `values` of a column of `data_type`."""
    return cardinality(registers([hash_value(v, data_type) for v in values], log2m), log2m)
