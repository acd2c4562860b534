#include "plan.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace tsnap {

static const size_t kDtypeSize[TSNAP_DTYPE_COUNT] = {1, 1, 2, 4, 8, 2, 2, 4, 8, 1, 1, 1, 1, 1};

size_t dtype_size(int dt) {
    if (dt < 0 || dt >= TSNAP_DTYPE_COUNT) return 0;
    return kDtypeSize[dt];
}

static bool is_float(int dt) { return dt == TSNAP_F16 || dt == TSNAP_BF16 || dt == TSNAP_F32 || dt == TSNAP_F64; }

static bool is_quant(int dt) { return dt == TSNAP_QINT8 || dt == TSNAP_QUINT8; }

bool cast_supported(int s, int d) {
    if (s == d) return !is_quant(s);  // quantised wire elements only exist as the product of a quantising save
    if (is_quant(d)) return is_float(s);  // the quantisers take the four wide floats only
    return (is_float(s) || is_fp8_dtype(s)) && (is_float(d) || is_fp8_dtype(d));
}

// TSNAP_QSCHEME_PER_CHANNEL: float -> int8 or scaled float8 on save, and back on restore
static bool per_channel_narrow(int dt) { return is_quant(dt) || is_fp8_dtype(uint32_t(dt)); }
static bool per_channel_supported(int s, int d) { return (is_float(s) && per_channel_narrow(d)) || (per_channel_narrow(s) && is_float(d)); }

static inline uint64_t lowbit(uint64_t x) { return x & (~x + 1); }

struct Dim {
    int64_t size, ss, ds;  // strides in bytes
};

static bool tile_fits_u32(const Member& m, int a, int b, uint32_t esz) {
    const uint32_t sa = transpose_side_a(esz), sb = transpose_side_b(esz);
    long double n = 1;
    for (uint32_t i = 0; i < m.nouter; ++i)
        n *= int(i) == a ? (long double)((uint64_t(m.osize[i]) + sa - 1) / sa) : int(i) == b ? (long double)((uint64_t(m.osize[i]) + sb - 1) / sb) : (long double)m.osize[i];
    return n < 4.0e9L;
}

int normalize_copy(const tsnap_copy_desc& d, uint64_t wire_base, bool allow_bulk, NormalizedCopy* out,
                   std::string* err) {
    out->n = 0;
    out->src_space = d.src_space;
    out->dst_space = d.dst_space;
    auto fail = [&](int code, const std::string& msg) {
        if (err) *err = msg;
        return code;
    };
    if (d.ndim < 0 || d.ndim > TSNAP_MAX_DIMS) return fail(TSNAP_EINVAL, "ndim out of range");
    const size_t es = dtype_size(d.src_dtype), ed = dtype_size(d.dst_dtype);
    if (es == 0 || ed == 0) return fail(TSNAP_EINVAL, "unknown dtype");
    if (d.src_space < 0 || d.src_space > TSNAP_SPACE_WIRE || d.dst_space < 0 || d.dst_space > TSNAP_SPACE_WIRE)
        return fail(TSNAP_EINVAL, "unknown address space");
    if (d.src_space == TSNAP_SPACE_WIRE && d.dst_space == TSNAP_SPACE_WIRE)
        return fail(TSNAP_EINVAL, "wire-to-wire copies are not a thing");
    const bool cast = d.src_dtype != d.dst_dtype;
    if (d.reserved != TSNAP_QSCHEME_PER_TENSOR && d.reserved != TSNAP_QSCHEME_PER_CHANNEL)
        return fail(TSNAP_EINVAL, "unknown quantisation scheme in tsnap_copy_desc.reserved");
    const bool per_channel = d.reserved == TSNAP_QSCHEME_PER_CHANNEL;
    if (per_channel ? !per_channel_supported(d.src_dtype, d.dst_dtype) : !cast_supported(d.src_dtype, d.dst_dtype))
        return fail(TSNAP_EUNSUP, "unsupported dtype conversion");
    const bool quant = is_quant(d.dst_dtype);
    if (!per_channel && quant && (d.dst_space != TSNAP_SPACE_WIRE || !(d.q_scale > 0)))
        return fail(TSNAP_EINVAL, "quantising copies need a WIRE destination and q_scale > 0");
    const bool pc_save = per_channel && per_channel_narrow(d.dst_dtype);  // a per-channel save (else a restore)
    if (per_channel && (pc_save ? d.dst_space : d.src_space) != TSNAP_SPACE_WIRE)
        return fail(TSNAP_EINVAL, "per-channel copies keep the quantised side in WIRE space");

    // logical shape; C-contiguous element strides for a WIRE destination
    int64_t cstride[TSNAP_MAX_DIMS];
    {
        int64_t acc = 1;
        for (int i = d.ndim - 1; i >= 0; --i) {
            if (d.sizes[i] < 0) return fail(TSNAP_EINVAL, "negative size");
            cstride[i] = acc;
            acc *= d.sizes[i];
        }
    }
    uint64_t numel = 1;
    for (int i = 0; i < d.ndim; ++i) numel *= uint64_t(d.sizes[i]);
    if (per_channel) {
        // the record is the caller's: read it once, check it against the descriptor, keep absolute addresses
        if (d.q_zero_point == 0) return fail(TSNAP_EINVAL, "per-channel descriptor without a tsnap_qchannel record");
        tsnap_qchannel r;
        std::memcpy(&r, reinterpret_cast<const void*>(uintptr_t(d.q_zero_point)), sizeof(r));
        if (r.channels <= 0 || r.inner <= 0 || r.channels > (int64_t(1) << 40) || r.inner > (int64_t(1) << 50))
            return fail(TSNAP_EINVAL, "tsnap_qchannel: channels and inner must be positive");
        const uint64_t period = uint64_t(r.channels) * uint64_t(r.inner);
        if (r.params_addr < r.body_addr || (r.params_addr - r.body_addr) % period != 0)
            return fail(TSNAP_EINVAL, "tsnap_qchannel: the body is not a whole number of channels x inner elements");
        if (pc_save) {
            if (r.body_addr < 8 || d.dst_addr != r.body_addr || r.params_addr != r.body_addr + numel)
                return fail(TSNAP_EINVAL, "tsnap_qchannel: a per-channel save writes the whole piece: header at body - 8, "
                                          "body at dst_addr, parameters right behind it");
            if (r.axis < 0 || r.axis >= d.ndim) return fail(TSNAP_EINVAL, "tsnap_qchannel: axis out of range");
        } else if (numel) {
            uint64_t last = d.src_addr;
            for (int i = 0; i < d.ndim; ++i) last += uint64_t(d.sizes[i] - 1) * uint64_t(d.src_strides[i]);
            if (d.src_addr < r.body_addr || last >= r.params_addr)
                return fail(TSNAP_EINVAL, "tsnap_qchannel: the member reads outside the piece's body");
        }
        out->qc.body = r.body_addr + wire_base;
        out->qc.params = r.params_addr + wire_base;
        out->qc.channels = uint64_t(r.channels);
        out->qc.inner = uint64_t(r.inner);
        out->qc.axis = r.axis;
        out->qc.save = pc_save ? 1 : 0;
        out->qc.param_bytes = is_fp8_dtype(uint32_t(pc_save ? d.dst_dtype : d.src_dtype)) ? 4 : 16;
    }
    if (numel == 0) return TSNAP_OK;

    Dim dims[TSNAP_MAX_DIMS];
    int nd = 0;
    for (int i = 0; i < d.ndim; ++i) {
        if (d.sizes[i] == 1) continue;
        Dim x;
        x.size = d.sizes[i];
        int64_t ss = d.src_strides[i];
        int64_t ds = d.dst_space == TSNAP_SPACE_WIRE ? cstride[i] : d.dst_strides[i];
        if (ss < 0 || ds < 0) return fail(TSNAP_EINVAL, "negative strides are not supported");
        if (ds == 0) return fail(TSNAP_EINVAL, "destination stride 0 with size > 1 (overlapping writes)");
        x.ss = ss * int64_t(es);
        x.ds = ds * int64_t(ed);
        // merge with the previous (outer) dim when both sides are dense across the boundary
        if (nd > 0 && dims[nd - 1].ss == x.ss * x.size && dims[nd - 1].ds == x.ds * x.size) {
            dims[nd - 1].size *= x.size;
            dims[nd - 1].ss = x.ss;
            dims[nd - 1].ds = x.ds;
        } else {
            dims[nd++] = x;
        }
    }

    Member m;
    std::memset(&m, 0, sizeof(m));
    m.src = d.src_addr + (d.src_space == TSNAP_SPACE_WIRE ? wire_base : 0);
    m.dst = d.dst_addr + (d.dst_space == TSNAP_SPACE_WIRE ? wire_base : 0);
    m.src_dtype = uint32_t(d.src_dtype);
    m.dst_dtype = uint32_t(d.dst_dtype);
    m.src_esz = uint32_t(es);
    m.dst_esz = uint32_t(ed);
    m.bytes = numel * ed;

    if (cast) {
        m.mode = kModeCast;
        m.unit = uint32_t(ed);
        if (quant && !per_channel) {
            m.q_scale = d.q_scale;
            m.q_zero_point = d.q_zero_point;
            m.shift = 1;  // append [scale][zero_point] behind the payload
        }
        if (nd > 0 && dims[nd - 1].ss == int64_t(es) && dims[nd - 1].ds == int64_t(ed)) {
            m.inner = uint64_t(dims[nd - 1].size);
            --nd;
        } else {
            m.inner = 1;
        }
    } else {
        if (nd > 0 && dims[nd - 1].ss == int64_t(es) && dims[nd - 1].ds == int64_t(ed)) {
            m.inner = uint64_t(dims[nd - 1].size) * ed;
            --nd;
        } else {
            m.inner = ed;
        }
    }
    if (nd > kMaxOuter) return fail(TSNAP_EUNSUP, "too many non-mergeable dimensions");
    m.nouter = uint32_t(nd);
    for (int i = 0; i < nd; ++i) {
        m.osize[i] = dims[i].size;
        m.sstride[i] = dims[i].ss;
        m.dstride[i] = dims[i].ds;
    }

    if (cast) {
        if (per_channel) {
            m.mode = out->qc.param_bytes == 4 ? kModeQChannelFp8 : kModeQChannel;
            m.shift = 0;
        }
        out->m[0] = m;
        out->n = 1;
        return TSNAP_OK;
    }
    if (nd == 0) {
        // one dense run on both sides
        const bool device_copy = d.src_space != TSNAP_SPACE_HOST && d.dst_space != TSNAP_SPACE_HOST;
        if (allow_bulk && device_copy && (m.src & 15) == 0 && (m.dst & 15) == 0 && m.bytes >= kBulkMin) {
            const uint64_t body = m.bytes & ~uint64_t(15);
            Member b = m;
            b.mode = kModeBulk;
            b.bytes = body;
            b.inner = body;
            b.unit = 16;
            out->m[out->n++] = b;
            if (m.bytes != body) {
                Member t = m;
                t.mode = kModeContig;
                t.src += body;
                t.dst += body;
                t.bytes = m.bytes - body;
                t.inner = t.bytes;
                t.shift = uint32_t(t.dst & 15);
                t.unit = 1;
                out->m[out->n++] = t;
            }
            return TSNAP_OK;
        }
        m.mode = kModeContig;
        m.shift = uint32_t(m.dst & 15);
        m.unit = uint32_t(lowbit(16 | ((m.src - m.dst) & 15)));  // widest load granule that is aligned whenever dst is
        out->m[0] = m;
        out->n = 1;
        return TSNAP_OK;
    }
    if (m.inner == ed && nd >= 2 && nd <= kMaxOuter) {
        // No run is contiguous on both sides.  If the source is unit-stride along one dim and the destination along
        // another (t(), permute of a dense tensor), tile over those two dims through shared memory.
        int a = -1, b = -1;
        for (int i = 0; i < nd; ++i) {
            if (m.sstride[i] == int64_t(es) && a < 0) a = i;
            if (m.dstride[i] == int64_t(ed) && b < 0) b = i;
        }
        bool aligned = (m.src % es) == 0 && (m.dst % ed) == 0;
        for (int i = 0; i < nd; ++i) aligned = aligned && (uint64_t(m.sstride[i]) % es) == 0 && (uint64_t(m.dstride[i]) % ed) == 0;
        const bool device_copy = d.src_space != TSNAP_SPACE_HOST && d.dst_space != TSNAP_SPACE_HOST;
        if (device_copy && aligned && a >= 0 && b >= 0 && a != b && m.osize[a] >= 16 && m.osize[b] >= 16 && tile_fits_u32(m, a, b, uint32_t(ed))) {
            m.mode = kModeTranspose;
            m.unit = uint32_t(ed);
            m.shift = uint32_t(a) | (uint32_t(b) << 8);
            out->m[0] = m;
            out->n = 1;
            return TSNAP_OK;
        }
    }
    m.mode = kModeStrided;
    uint64_t bits = 16 | m.inner | m.src | m.dst;
    for (int i = 0; i < nd; ++i) bits |= uint64_t(m.sstride[i]) | uint64_t(m.dstride[i]);
    m.unit = uint32_t(lowbit(bits));
    {
        // Column shards / narrow on dim != 0 of wide tables (T:io_preparers/sharded_tensor.py:76, torchrec COLUMN_WISE)
        // and reshard boxes have long 16 B-aligned runs: those go to the copy engine run by run.
        const bool device_copy = d.src_space != TSNAP_SPACE_HOST && d.dst_space != TSNAP_SPACE_HOST;
        if (allow_bulk && device_copy && m.unit == 16 && m.inner >= kRowsMinRun) {
            m.mode = kModeRows;
            // is a side laid out run after run (the wire side always is)?
            uint64_t accs = m.inner, accd = m.inner;
            bool sd = true, dd = true;
            for (int i = nd - 1; i >= 0; --i) {
                sd = sd && uint64_t(m.sstride[i]) == accs;
                dd = dd && uint64_t(m.dstride[i]) == accd;
                accs *= uint64_t(m.osize[i]);
                accd *= uint64_t(m.osize[i]);
            }
            m.shift = (sd ? kRowsSrcDense : 0) | (dd ? kRowsDstDense : 0);
        }
    }
    out->m[0] = m;
    out->n = 1;
    return TSNAP_OK;
}

// ---- host execution -------------------------------------------------------------------------------------

void host_copy_range(const Member& m, uint64_t lo, uint64_t hi) {
    if (hi > m.bytes) hi = m.bytes;
    if (lo >= hi) return;
    const char* src = reinterpret_cast<const char*>(uintptr_t(m.src));
    char* dst = reinterpret_cast<char*>(uintptr_t(m.dst));
    if (m.mode == kModeBulk || m.mode == kModeContig) {
        std::memcpy(dst + lo, src + lo, hi - lo);
        return;
    }
    if (m.mode == kModeStrided || m.mode == kModeRows || m.mode == kModeTranspose) {
        uint64_t pos = lo;
        while (pos < hi) {
            const uint64_t row = pos / m.inner, col = pos % m.inner;
            uint64_t n = m.inner - col;
            if (n > hi - pos) n = hi - pos;
            int64_t so, dofs;
            outer_offsets(m, row, &so, &dofs);
            std::memcpy(dst + dofs + col, src + so + col, n);
            pos += n;
        }
        return;
    }
    // cast: lo/hi are dst bytes, multiples of the dst element size by construction.  Elements are read and written
    // byte by byte (aligned = false): host pointers may sit at any alignment, and the compiler merges the bytes.
    const uint64_t e0 = lo / m.dst_esz, e1 = hi / m.dst_esz;
    const bool quant = m.dst_dtype == TSNAP_QINT8 || m.dst_dtype == TSNAP_QUINT8;
    for (uint64_t e = e0; e < e1; ++e) {
        const uint64_t row = e / m.inner, col = e % m.inner;
        int64_t so, dofs;
        outer_offsets(m, row, &so, &dofs);
        if (quant) {
            const float x = load_f32(src + so + col * m.src_esz, m.src_dtype, false);
            reinterpret_cast<uint8_t*>(dst + dofs)[col] = quantize_elem(x, m.q_scale, m.q_zero_point, m.dst_dtype == TSNAP_QINT8);
        } else {
            convert_store(dst + dofs + col * m.dst_esz, m.dst_dtype, src + so + col * m.src_esz, m.src_dtype, false, false);
        }
    }
    if (quant && (m.shift & 1) && hi == m.bytes) {
        std::memcpy(dst + m.bytes, &m.q_scale, 8);
        std::memcpy(dst + m.bytes + 8, &m.q_zero_point, 8);
    }
}

// ---- per-channel quantisation on the host ------------------------------------------------------------------
// The three passes of the device (statistics, parameters, quantising pack) in one sequential sweep each, with the same
// rules: the element as fp32, channel keys that start at 0, the parameters of qparams_of, torch's CPU quantiser.  A
// float8 wire (kModeQChannelFp8) takes fp8_scale_of, fp8_quantize and fp8_dequantize instead, with f32 scales.
int host_qchannel(const Member& m, const QChannel& q, std::string* err) {
    const char* src = reinterpret_cast<const char*>(uintptr_t(m.src));
    char* dst = reinterpret_cast<char*>(uintptr_t(m.dst));
    const uint64_t n = m.bytes / m.dst_esz;
    char* params = reinterpret_cast<char*>(uintptr_t(q.params));
    auto channel = [&](uint64_t wire_addr) { return ((wire_addr - q.body) / q.inner) % q.channels; };
    const bool fp8 = m.mode == kModeQChannelFp8;
    const uint32_t wire_dt = q.save ? m.dst_dtype : m.src_dtype;
    const bool is_signed = wire_dt == TSNAP_QINT8;
    if (!q.save) {
        for (uint64_t e = 0; e < n; ++e) {
            const uint64_t row = e / m.inner, col = e % m.inner;
            int64_t so, dofs;
            outer_offsets(m, row, &so, &dofs);
            const uint64_t a = m.src + uint64_t(so) + col;
            const uint64_t c = channel(a);
            const uint8_t raw = *reinterpret_cast<const uint8_t*>(uintptr_t(a));
            float f;
            if (fp8) {
                float s;
                std::memcpy(&s, params + 4 * c, 4);
                f = fp8_dequantize(raw, wire_dt, s);
            } else {
                double scale;
                int64_t zp;
                std::memcpy(&scale, params + 8 * c, 8);
                std::memcpy(&zp, params + 8 * (q.channels + c), 8);
                f = dequantize(raw, is_signed, zp, scale);
            }
            store_f32(dst + dofs + col * m.dst_esz, m.dst_dtype, f, false);
        }
        return TSNAP_OK;
    }
    std::vector<int32_t> kmin(q.channels, 0), kmax(q.channels, 0);
    for (uint64_t e = 0; e < n; ++e) {
        const uint64_t row = e / m.inner, col = e % m.inner;
        int64_t so, dofs;
        outer_offsets(m, row, &so, &dofs);
        const int32_t k = qkey(load_f32(src + so + col * m.src_esz, m.src_dtype, false));
        const uint64_t c = channel(m.dst + uint64_t(dofs) + col);
        kmin[c] = std::min(kmin[c], k);
        kmax[c] = std::max(kmax[c], k);
    }
    std::vector<double> scale(fp8 ? 0 : q.channels);
    std::vector<int64_t> zp(fp8 ? 0 : q.channels);
    std::vector<float> fp8_scale(fp8 ? q.channels : 0);
    for (uint64_t c = 0; c < q.channels; ++c) {
        if (fp8 ? !fp8_scale_of(kmin[c], kmax[c], wire_dt, &fp8_scale[c]) : !qparams_of(kmin[c], kmax[c], is_signed, &scale[c], &zp[c])) {
            if (err) *err = "per-channel quantisation: channel " + std::to_string(c) + " holds a NaN or Inf";
            return TSNAP_EINVAL;
        }
    }
    std::memcpy(reinterpret_cast<char*>(uintptr_t(q.body)) - 8, &q.axis, 8);
    if (fp8) {
        std::memcpy(params, fp8_scale.data(), 4 * q.channels);
    } else {
        std::memcpy(params, scale.data(), 8 * q.channels);
        std::memcpy(params + 8 * q.channels, zp.data(), 8 * q.channels);
    }
    for (uint64_t e = 0; e < n; ++e) {
        const uint64_t row = e / m.inner, col = e % m.inner;
        int64_t so, dofs;
        outer_offsets(m, row, &so, &dofs);
        const float x = load_f32(src + so + col * m.src_esz, m.src_dtype, false);
        const uint64_t c = channel(m.dst + uint64_t(dofs) + col);
        reinterpret_cast<uint8_t*>(dst + dofs)[col] = fp8 ? fp8_quantize(x, fp8_scale[c], wire_dt) : quantize_elem(x, scale[c], zp[c], is_signed);
    }
    return TSNAP_OK;
}

int host_copy_all(const NormalizedCopy& nc, std::string* err) {
    if (nc.n == 1 && qchannel_mode(nc.m[0].mode)) return host_qchannel(nc.m[0], nc.qc, err);
    for (int k = 0; k < nc.n; ++k) host_copy_range(nc.m[k], 0, nc.m[k].bytes);
    return TSNAP_OK;
}

}  // namespace tsnap
