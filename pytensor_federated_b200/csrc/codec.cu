// Native proto3 codec for the ArraysToArrays messages (host code only).
//
// InputArrays / OutputArrays = { repeated npproto.ndarray items = 1; string uuid = 2; }
// npproto.ndarray            = { bytes data = 1; string dtype = 2; repeated int64 shape = 3 [packed];
//                                repeated int64 strides = 4 [packed]; }
// Schema: protobufs/service.proto:6-19, npproto/ndarray.proto:7-12.  The Python
// implementation (pytensor_federated_b200/_pb.py, rpc.py) is the fallback and the oracle: both must
// produce identical bytes (tests/test_native_codec.py).  One call encodes a whole message into a
// caller-provided buffer with a single memcpy per array; decoding returns offsets so that NumPy can
// build zero-copy views over the received buffer.
#include <cstdint>
#include <cstring>

namespace {

inline int varint_size(uint64_t v) {
    int n = 1;
    while (v > 0x7F) { v >>= 7; ++n; }
    return n;
}
inline unsigned char* put_varint(unsigned char* p, uint64_t v) {
    while (v > 0x7F) { *p++ = (unsigned char)((v & 0x7F) | 0x80); v >>= 7; }
    *p++ = (unsigned char)v;
    return p;
}
inline bool get_varint(const unsigned char*& p, const unsigned char* end, uint64_t& v) {
    v = 0;
    for (int shift = 0; shift < 70; shift += 7) {
        if (p >= end) return false;
        const unsigned char b = *p++;
        v |= (uint64_t)(b & 0x7F) << shift;
        if (!(b & 0x80)) return true;
    }
    return false;
}
inline long long packed_size(const long long* vals, int n) {
    long long s = 0;
    for (int i = 0; i < n; ++i) s += varint_size((uint64_t)vals[i]);
    return s;
}
long long ndarray_size(long long nbytes, long long dtype_len, const long long* shape, const long long* strides, int ndim) {
    long long s = 0;
    if (nbytes > 0) s += 1 + varint_size((uint64_t)nbytes) + nbytes;
    if (dtype_len > 0) s += 1 + varint_size((uint64_t)dtype_len) + dtype_len;
    if (ndim > 0) {
        const long long ps = packed_size(shape, ndim), pt = packed_size(strides, ndim);
        s += 1 + varint_size((uint64_t)ps) + ps;
        s += 1 + varint_size((uint64_t)pt) + pt;
    }
    return s;
}

}  // namespace

extern "C" {

struct B200PbItem {
    long long data_off, data_len, dtype_off, dtype_len;
    int ndim, n_strides;
    long long shape[16];
    long long strides[16];
};

// Returns the encoded size.  Writes the message when cap >= size (otherwise nothing is written).
long long b200_pb_encode_arrays(int n_items, const void* const* data, const long long* nbytes, const char* const* dtypes,
                                const int* ndims, const long long* shapes, const long long* strides, const char* uuid,
                                unsigned char* out, long long cap) {
    long long total = 0;
    int off = 0;
    for (int i = 0; i < n_items; ++i) {
        const long long item = ndarray_size(nbytes[i], (long long)strlen(dtypes[i]), shapes + off, strides + off, ndims[i]);
        total += 1 + varint_size((uint64_t)item) + item;
        off += ndims[i];
    }
    const long long uuid_len = uuid ? (long long)strlen(uuid) : 0;
    if (uuid_len > 0) total += 1 + varint_size((uint64_t)uuid_len) + uuid_len;
    if (!out || cap < total) return total;

    unsigned char* p = out;
    off = 0;
    for (int i = 0; i < n_items; ++i) {
        const long long dlen = (long long)strlen(dtypes[i]);
        const long long item = ndarray_size(nbytes[i], dlen, shapes + off, strides + off, ndims[i]);
        *p++ = 0x0A;
        p = put_varint(p, (uint64_t)item);
        if (nbytes[i] > 0) {
            *p++ = 0x0A;
            p = put_varint(p, (uint64_t)nbytes[i]);
            memcpy(p, data[i], (size_t)nbytes[i]);
            p += nbytes[i];
        }
        if (dlen > 0) {
            *p++ = 0x12;
            p = put_varint(p, (uint64_t)dlen);
            memcpy(p, dtypes[i], (size_t)dlen);
            p += dlen;
        }
        if (ndims[i] > 0) {
            *p++ = 0x1A;
            p = put_varint(p, (uint64_t)packed_size(shapes + off, ndims[i]));
            for (int d = 0; d < ndims[i]; ++d) p = put_varint(p, (uint64_t)shapes[off + d]);
            *p++ = 0x22;
            p = put_varint(p, (uint64_t)packed_size(strides + off, ndims[i]));
            for (int d = 0; d < ndims[i]; ++d) p = put_varint(p, (uint64_t)strides[off + d]);
        }
        off += ndims[i];
    }
    if (uuid_len > 0) {
        *p++ = 0x12;
        p = put_varint(p, (uint64_t)uuid_len);
        memcpy(p, uuid, (size_t)uuid_len);
        p += uuid_len;
    }
    return (long long)(p - out);
}

static bool skip_field(const unsigned char*& p, const unsigned char* end, int wt) {
    uint64_t v;
    switch (wt) {
        case 0: return get_varint(p, end, v);
        case 1: if (end - p < 8) return false; p += 8; return true;
        case 2: if (!get_varint(p, end, v) || (uint64_t)(end - p) < v) return false; p += v; return true;
        case 5: if (end - p < 4) return false; p += 4; return true;
        default: return false;
    }
}

static bool parse_int64s(const unsigned char*& p, const unsigned char* end, int wt, long long* dst, int& count, int cap) {
    uint64_t v;
    if (wt == 0) {  // unpacked element
        if (!get_varint(p, end, v)) return false;
        if (count < cap) dst[count] = (long long)v;
        ++count;
        return true;
    }
    if (wt != 2) return false;
    uint64_t len;
    if (!get_varint(p, end, len) || (uint64_t)(end - p) < len) return false;
    const unsigned char* e = p + len;
    while (p < e) {
        if (!get_varint(p, e, v)) return false;
        if (count < cap) dst[count] = (long long)v;
        ++count;
    }
    return true;
}

// Returns the number of items (may exceed max_items: call again with a larger array), -1 on malformed
// input, or -2 for a well-formed message this fast path does not cover (an array with more than 16
// dimensions): the caller falls back to the general decoder.  Offsets are relative to `buf`.
long long b200_pb_decode_arrays(const unsigned char* buf, long long len, B200PbItem* items, int max_items,
                                long long* uuid_off, long long* uuid_len) {
    const unsigned char* p = buf;
    const unsigned char* end = buf + len;
    long long n = 0;
    *uuid_off = 0;
    *uuid_len = 0;
    while (p < end) {
        uint64_t key;
        if (!get_varint(p, end, key)) return -1;
        const int field = (int)(key >> 3), wt = (int)(key & 7);
        if (field == 1 && wt == 2) {
            uint64_t ilen;
            if (!get_varint(p, end, ilen) || (uint64_t)(end - p) < ilen) return -1;
            const unsigned char* q = p;
            const unsigned char* qe = p + ilen;
            B200PbItem it;
            memset(&it, 0, sizeof(it));
            while (q < qe) {
                uint64_t k2;
                if (!get_varint(q, qe, k2)) return -1;
                const int f2 = (int)(k2 >> 3), w2 = (int)(k2 & 7);
                if ((f2 == 1 || f2 == 2) && w2 == 2) {
                    uint64_t l2;
                    if (!get_varint(q, qe, l2) || (uint64_t)(qe - q) < l2) return -1;
                    if (f2 == 1) { it.data_off = q - buf; it.data_len = (long long)l2; }
                    else { it.dtype_off = q - buf; it.dtype_len = (long long)l2; }
                    q += l2;
                } else if (f2 == 3) {
                    if (!parse_int64s(q, qe, w2, it.shape, it.ndim, 16)) return -1;
                } else if (f2 == 4) {
                    if (!parse_int64s(q, qe, w2, it.strides, it.n_strides, 16)) return -1;
                } else if (!skip_field(q, qe, w2)) {
                    return -1;
                }
            }
            if (it.ndim > 16 || it.n_strides > 16) return -2;   // valid, but more dimensions than B200PbItem holds
            if (n < max_items) items[n] = it;
            ++n;
            p = qe;
        } else if (field == 2 && wt == 2) {
            uint64_t l;
            if (!get_varint(p, end, l) || (uint64_t)(end - p) < l) return -1;
            *uuid_off = p - buf;
            *uuid_len = (long long)l;
            p += l;
        } else if (!skip_field(p, end, wt)) {
            return -1;
        }
    }
    return n;
}

}  // extern "C"
