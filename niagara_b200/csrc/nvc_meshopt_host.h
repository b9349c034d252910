// nvc_meshopt_host.h — the host decoders of the meshopt codecs, inline so that every translation unit that decodes links on its
// own: the scene-cache reader (nvc_scene_cache.cpp), the glTF importer (nvc_gltf.cpp, EXT_ / KHR_meshopt_compression buffer
// views) and the exported decoders (nvc_meshopt_decode.cpp).  Host only; the .cu files never include it.  Build with
// -ffp-contract=off: the vertex filters must round every operation as the reference's SSE2 build does.
//
// Formats (meshoptimizer v1.0, extern/meshoptimizer/src/vertexcodec.cpp, indexcodec.cpp, vertexfilter.cpp — restated, not
// copied):
//
// VERTEX stream   [0xa0 | version] blocks... tail
//   tail  = the last max(tail, 24 (v1) / 32 (v0)) bytes; its final `stride` (+ stride/4 for v1) bytes hold the
//           baseline vertex and, for v1, one channel byte per 4-byte group
//   block = min(256, (8192 / stride) & ~15) vertices; [v1: stride/4 control bytes]; then per 4-byte group its four
//           byte planes, each: control 3 = `count` literal bytes, 2 = all zero, 0/1 = byte groups
//   byte groups: 2-bit selector per 16 values ((groups + 3) / 4 header bytes) into the width table
//           v0 {0,2,4,8}, v1 control 0 {0,1,2,4}, control 1 {1,2,4,8}; width 0 = zeros, 8 = 16 literals, else 16 packed
//           values (1-bit: LSB first, 2/4-bit: MSB first) where the all-ones value means "next escape byte"
//   deltas per 4-byte group by channel & 3: 0 = per byte zigzag delta, 1 = per 16-bit zigzag delta,
//           2 = 32-bit xor with the previous value after rotating left by (32 - (channel >> 4)) & 31 (vcodec::delta_term)
//
// INDEX stream    [0xe0 | version] one code byte per triangle, data bytes, 16-byte aux table at the very end
//   code < 0xf0 : high nibble = edge FIFO slot (a, b), low nibble = c: 0 next new vertex, 1..12 (v1) / 1..14 (v0)
//                 vertex FIFO slot, 13 / 14 (v1) = last -/+ 1, 15 = explicit zigzag varint delta from `last`
//   0xf0..0xfd  : restart, (b, c) slots from aux[code & 15]; a = next new vertex
//   0xfe / 0xff : restart with an explicit aux byte (0xff: a explicit too); aux == 0 resets the vertex counter
//
// INDEX SEQUENCE  [0xd0 | version] one varint per index, then 4 zero bytes
//   varint v (7 bits per byte, low group first, at most 5 bytes): bit 0 picks one of two baselines, v >> 1 is a zigzag
//   delta from that baseline; the decoded index becomes the baseline's new value.  The varints must end exactly where the
//   4-byte tail starts.  Versions 0 and 1 decode alike.
//
// VERTEX FILTERS  applied in place to a decoded ATTRIBUTES view, four elements at a time as the SSE2 build does (the last
//   count % 4 elements through a zeroed 4-element temporary); float -> int conversions round to nearest even, NaN and
//   out-of-range values give 0x80000000 (cvtps2dq)
//   OCTAHEDRAL  stride 4: signed 8-bit x, y, z, w kept; stride 8: signed 16-bit x, y, 15-bit z, w kept.  z -= |x| + |y|;
//               for z < 0, x and y move |z| towards zero; the vector is scaled to length 127 by rsqrtps (stride 4) or to
//               32767 by a division by sqrt (stride 8)
//   QUATERNION  stride 8: three signed 16-bit components and a fourth one whose low 2 bits name the dropped component
//               and whose value | 3 is the fixed-point scale; the dropped one is sqrt(2 s^2 - |xyz|^2); stored w, x, y, z
//               then rotated left by 16 bits per the named index
//   EXPONENTIAL any stride, per 32-bit word: 2^(signed high byte) * (signed low 24 bits) as a float
//   COLOR       stride 4 / 8: Y, Co, Cg and alpha whose highest set bit gives the bit count; RGBA scaled to 255 by rcpps
//               (stride 4) or to 65535 by a division (stride 8)
//   rsqrtps and rcpps are approximations whose bits the CPU defines; on x86 the filters execute those instructions, so the
//   output equals the reference's decoder run on the same host.  Elsewhere they use the exact 1 / sqrt and 1 / x.
#pragma once

#include "nvc_meshopt_format.h"

#include <math.h>
#include <string.h>

#if defined(__SSE2__) || defined(_M_X64)
#include <emmintrin.h>
#define NVC_FILTER_SSE 1
#endif

namespace nvc
{
namespace mhost
{

struct ByteReader
{
	const uint8_t* at;
	const uint8_t* end;
	bool take(size_t n, const uint8_t*& out)
	{
		if (size_t(end - at) < n)
			return false;
		out = at;
		at += n;
		return true;
	}
};

// One byte plane of `count` values from r: control 3 = literals, 2 = zeros, else the selector header and its groups.
// `group(g, width, bytes)` is called for every group of 16 values with the group_bytes(bytes, width) bytes it occupies;
// false when the plane runs past r.end.  The decoder unpacks in `group`, the walk only measures.
template <typename Group>
inline bool walk_plane(ByteReader& r, int control, int version, uint32_t count, Group&& group)
{
	const uint8_t* bytes;
	if (control == 3)
		return r.take(count, bytes);
	if (control == 2)
		return true;
	const uint32_t groups = (count + 15u) / 16u;
	const uint8_t* selectors;
	if (!r.take(vcodec::selector_bytes(groups), selectors))
		return false;
	for (uint32_t g = 0; g < groups; ++g)
	{
		const int width = vcodec::group_width(version, control, (selectors[g / 4] >> ((g % 4) * 2)) & 3u);
		const size_t packed = width == 8 ? 16 : size_t(2 * width); // readable before the escapes can be counted
		if (size_t(r.end - r.at) < packed || !r.take(vcodec::group_bytes(r.at, width), bytes))
			return false;
		group(g, width, bytes);
	}
	return true;
}

inline bool read_plane(ByteReader& r, int control, int version, uint32_t count, uint8_t* out /* room for count rounded up to 16 */)
{
	if (control == 3 || control == 2)
	{
		const uint8_t* lit = r.at;
		if (!walk_plane(r, control, version, count, [](uint32_t, int, const uint8_t*) {}))
			return false;
		if (control == 3)
			memcpy(out, lit, count);
		else
			memset(out, 0, count);
		return true;
	}
	return walk_plane(r, control, version, count, [&](uint32_t g, int width, const uint8_t* bytes) {
		if (width == 0)
			memset(out + g * 16, 0, 16);
		else if (width == 8)
			memcpy(out + g * 16, bytes, 16);
		else
			vcodec::unpack_group(bytes, width, out + g * 16);
	});
}

// The parts of a vertex stream around its blocks: the version, the baseline vertex and (v1) the channel bytes in the
// tail, and the byte range the blocks must fill exactly.
struct VertexStream
{
	int version;
	const uint8_t* baseline;
	const uint8_t* channels; // nullptr for v0 (channel 0 everywhere)
	ByteReader blocks;
};

inline int open_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t stride, VertexStream& out)
{
	if (stride == 0 || stride > 256 || stride % 4 != 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (stream_size < 1 || (stream[0] & 0xf0) != 0xa0)
		return NVC_ERROR_CORRUPT;
	const int version = stream[0] & 0x0f;
	if (version > 1)
		return NVC_ERROR_UNSUPPORTED;
	const size_t tail = stride + (version == 0 ? 0 : stride / 4);
	const size_t tail_min = version == 0 ? 32 : 24;
	const size_t tail_padded = tail < tail_min ? tail_min : tail;
	if (stream_size - 1 < tail_padded)
		return NVC_ERROR_CORRUPT;
	out.version = version;
	out.baseline = stream + stream_size - tail;
	out.channels = version == 0 ? nullptr : stream + stream_size - tail + stride;
	out.blocks = { stream + 1, stream + stream_size - tail_padded };
	return NVC_OK;
}

// varint of at most 5 bytes, 7 bits per byte, low group first
inline bool read_varint(ByteReader& r, uint32_t& value)
{
	value = 0;
	for (int i = 0; i < 5; ++i)
	{
		const uint8_t* b;
		if (!r.take(1, b))
			return false;
		value |= uint32_t(*b & 127u) << (7 * i);
		if (*b < 128)
			break;
	}
	return true;
}

inline bool read_varint_delta(ByteReader& r, uint32_t& last)
{
	uint32_t value;
	if (!read_varint(r, value))
		return false;
	last += (value >> 1) ^ (0u - (value & 1u));
	return true;
}

inline void store_index(void* out, size_t i, uint32_t index_size, uint32_t value)
{
	if (index_size == 2)
		static_cast<uint16_t*>(out)[i] = uint16_t(value);
	else
		static_cast<uint32_t*>(out)[i] = value;
}

} // namespace mhost

// 0 ok, negative NvcStatus otherwise
inline int decode_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t vertex_count, uint32_t stride, uint8_t* out)
{
	mhost::VertexStream vs;
	int status = mhost::open_vertex_stream(stream, stream_size, stride, vs);
	if (status != NVC_OK)
		return status;
	const int version = vs.version;
	const uint8_t* channels = vs.channels;
	uint8_t previous[256];
	memcpy(previous, vs.baseline, stride);
	mhost::ByteReader& r = vs.blocks;
	const uint32_t per_block = vcodec::block_vertices(stride);

	uint8_t planes[4][256 + 16];
	for (uint32_t first = 0; first < vertex_count; first += per_block)
	{
		uint32_t count = vertex_count - first < per_block ? vertex_count - first : per_block;
		const uint8_t* control = nullptr;
		if (version != 0 && !r.take(stride / 4, control))
			return NVC_ERROR_CORRUPT;
		uint8_t* block = out + size_t(first) * stride;
		for (uint32_t k = 0; k < stride; k += 4)
		{
			uint32_t ctrl = control ? control[k / 4] : 0u;
			for (int j = 0; j < 4; ++j)
				if (!mhost::read_plane(r, int((ctrl >> (j * 2)) & 3u), version, count, planes[j]))
					return NVC_ERROR_CORRUPT;
			const uint32_t channel = channels ? channels[k / 4] : 0u;
			if ((channel & 3) == 3) // no delta rule
				return NVC_ERROR_CORRUPT;
			uint32_t p;
			memcpy(&p, previous + k, 4);
			for (uint32_t i = 0; i < count; ++i)
			{
				const uint32_t v = uint32_t(planes[0][i]) | (uint32_t(planes[1][i]) << 8) | (uint32_t(planes[2][i]) << 16) | (uint32_t(planes[3][i]) << 24);
				p = vcodec::combine(p, vcodec::delta_term(v, channel), channel);
				memcpy(block + size_t(i) * stride + k, &p, 4);
			}
		}
		memcpy(previous, block + size_t(count - 1) * stride, stride);
	}
	return r.at == r.end ? NVC_OK : NVC_ERROR_CORRUPT;
}

// Indexes a vertex stream for the device decoder (nvc_cache_decode.cuh) without decoding it: for every block the offset
// of its first byte from the start of the stream (block_start[blocks] = where the blocks end) and, for each of its
// `stride` byte planes in stream order, the plane's offset from the block's start.  Only sizes are read: control bytes,
// selector headers, and the escape counts of the packed groups.  Walks the structure decode_vertex_stream decodes and
// returns the status it returns on every stream, so a stream the walk accepts decodes without a check on the device.
// Strides up to 16 (a block then spans less than 2^16 bytes); streams under 4 GiB, NVC_ERROR_UNSUPPORTED otherwise.
inline int walk_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t vertex_count, uint32_t stride, uint32_t* block_start, uint16_t* plane_offset,
    VertexStreamTail* tail)
{
	if (stride > 16)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (stream_size > 0xffffffffull)
		return NVC_ERROR_UNSUPPORTED; // block starts are 32-bit offsets
	mhost::VertexStream vs;
	int status = mhost::open_vertex_stream(stream, stream_size, stride, vs);
	if (status != NVC_OK)
		return status;
	tail->version = vs.version;
	tail->baseline = vs.baseline;
	tail->channels = vs.channels;
	mhost::ByteReader& r = vs.blocks;
	const uint32_t per_block = vcodec::block_vertices(stride);
	auto nothing = [](uint32_t, int, const uint8_t*) {};
	uint32_t b = 0;
	for (uint32_t first = 0; first < vertex_count; first += per_block, ++b)
	{
		uint32_t count = vertex_count - first < per_block ? vertex_count - first : per_block;
		const uint8_t* block = r.at;
		block_start[b] = uint32_t(block - stream);
		const uint8_t* control = nullptr;
		if (vs.version != 0 && !r.take(stride / 4, control))
			return NVC_ERROR_CORRUPT;
		for (uint32_t q = 0; q < stride; ++q)
		{
			plane_offset[size_t(b) * stride + q] = uint16_t(r.at - block);
			uint32_t ctrl = control ? (control[q / 4] >> ((q % 4) * 2)) & 3u : 0u;
			if (!mhost::walk_plane(r, int(ctrl), vs.version, count, nothing))
				return NVC_ERROR_CORRUPT;
		}
		// decode_vertex_stream rejects a channel it has no delta for at the first block
		for (uint32_t k = 0; vs.channels && b == 0 && k < stride / 4; ++k)
			if ((vs.channels[k] & 3) == 3)
				return NVC_ERROR_CORRUPT;
	}
	block_start[b] = uint32_t(r.at - stream);
	return r.at == r.end ? NVC_OK : NVC_ERROR_CORRUPT;
}

// Data bytes of an index stream for icodec::decode_triangle: those between the code bytes and the aux table
struct IndexData
{
	mhost::ByteReader r;
	bool next(uint32_t& b)
	{
		const uint8_t* p;
		if (!r.take(1, p))
			return false;
		b = *p;
		return true;
	}
};

// The index codec's decoder state over concrete indices (icodec::decode_triangle)
struct IndexState
{
	using Value = uint32_t;
	icodec::Ring16 verts, edges_a, edges_b;
	uint32_t next = 0, last = 0;
	static uint32_t add(uint32_t v, uint32_t k) { return v + k; }
	static uint32_t zero() { return 0; }
	uint32_t vert(uint32_t n) const { return verts.back(n); }
	uint32_t edge_a(uint32_t n) const { return edges_a.back(n); }
	uint32_t edge_b(uint32_t n) const { return edges_b.back(n); }
	void put_vert(uint32_t v, bool advance) { verts.put(v, advance); }
	void put_edge(uint32_t a, uint32_t b)
	{
		edges_a.put(a);
		edges_b.put(b);
	}
};

// The header checks of an index stream of index_count indices: its version, or a negative NvcStatus
inline int open_index_stream(const uint8_t* stream, size_t stream_size, uint32_t index_count)
{
	if (index_count % 3 != 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (stream_size < size_t(1) + index_count / 3 + 16)
		return NVC_ERROR_CORRUPT;
	if ((stream[0] & 0xf0) != 0xe0)
		return NVC_ERROR_CORRUPT;
	const int version = stream[0] & 0x0f;
	return version > 1 ? NVC_ERROR_UNSUPPORTED : version;
}

// code < 0xf0 with c = low nibble: FIFO slots below this, then last -/+ 1 (v1) and the explicit varint
inline uint32_t index_direct_slots(int version)
{
	return version >= 1 ? 13u : 15u;
}

// The index codec into index_size (2 or 4) bytes per index; 16-bit outputs keep the low half of each index
inline int decode_index_buffer(const uint8_t* stream, size_t stream_size, uint32_t index_count, uint32_t index_size, void* out)
{
	if (index_size != 2 && index_size != 4)
		return NVC_ERROR_INVALID_ARGUMENT;
	const int version = open_index_stream(stream, stream_size, index_count);
	if (version < 0)
		return version;
	const uint32_t triangles = index_count / 3, direct_slots = index_direct_slots(version);
	const uint8_t* codes = stream + 1;
	const uint8_t* aux = stream + stream_size - 16;
	IndexData data = { { codes + triangles, aux } };
	IndexState s;
	for (uint32_t t = 0; t < triangles; ++t)
	{
		uint32_t corner[3];
		if (!icodec::decode_triangle(s, codes[t], aux, direct_slots, data, corner))
			return NVC_ERROR_CORRUPT;
		mhost::store_index(out, size_t(t) * 3 + 0, index_size, corner[0]);
		mhost::store_index(out, size_t(t) * 3 + 1, index_size, corner[1]);
		mhost::store_index(out, size_t(t) * 3 + 2, index_size, corner[2]);
	}
	return data.r.at == data.r.end ? NVC_OK : NVC_ERROR_CORRUPT;
}

// A decoder state that holds nothing: icodec::decode_triangle over it only consumes data bytes
struct IndexShape
{
	struct Value
	{
	};
	Value next, last;
	static Value add(Value, uint32_t) { return Value(); }
	static Value zero() { return Value(); }
	Value vert(uint32_t) const { return Value(); }
	Value edge_a(uint32_t) const { return Value(); }
	Value edge_b(uint32_t) const { return Value(); }
	void put_vert(Value, bool) {}
	void put_edge(Value, Value) {}
};

// A data source that counts the bytes the step reads: the first is `first`, every later one ends a varint
struct IndexTokenCounter
{
	uint32_t first, reads;
	bool next(uint32_t& b)
	{
		b = reads++ == 0 ? first : 0u;
		return true;
	}
};

// Skips `count` varints from `at`; false when one runs past `end` (icodec::read_varint's rule: a varint ends at its first
// byte below 128 or after its fifth byte)
inline bool skip_varints(const uint8_t*& at, const uint8_t* end, uint32_t count)
{
	for (; count; --count)
		for (int i = 0;; ++i)
		{
			if (at == end)
				return false;
			if (*at++ < 128u || i == 4)
				break;
		}
	return true;
}

// Cuts an index stream into chunks of `chunk` triangles for the device decoder (nvc_cache_decode.cuh) without decoding
// it: chunk_data[c] = the offset from the stream's start of the first data byte triangle c * chunk reads, for every
// chunk c.  Only code bytes, the aux bytes of 0xfe / 0xff and the ends of varints are read.  How many varints a triangle
// holds comes from the decoder's own step (icodec::decode_triangle over a state that holds nothing), tabled per code
// and per aux byte, and the walk reads the data bytes in the decoder's order, so it returns the status
// decode_index_buffer returns on every stream, and a stream it accepts decodes on the device without a check.  Returns
// the version (0 or 1), or a negative NvcStatus.
inline int walk_index_stream(const uint8_t* stream, size_t stream_size, uint32_t index_count, uint32_t chunk, uint64_t* chunk_data)
{
	const int version = open_index_stream(stream, stream_size, index_count);
	if (version < 0)
		return version;
	const uint32_t triangles = index_count / 3, direct_slots = index_direct_slots(version);
	const uint8_t* codes = stream + 1;
	const uint8_t* aux = stream + stream_size - 16;
	// varints of a triangle by its code (below 0xfe), and after the aux byte x of 0xfe / 0xff
	uint8_t varints[256], varints_after[2][256];
	IndexShape s;
	IndexShape::Value corner[3];
	for (uint32_t code = 0; code < 256; ++code)
	{
		IndexTokenCounter count = { 0, 0 };
		if (code < 0xfe)
			icodec::decode_triangle(s, code, aux, direct_slots, count, corner);
		varints[code] = uint8_t(count.reads);
	}
	for (uint32_t x = 0; x < 256; ++x)
		for (uint32_t k = 0; k < 2; ++k)
		{
			IndexTokenCounter count = { x, 0 };
			icodec::decode_triangle(s, 0xfe + k, aux, direct_slots, count, corner);
			varints_after[k][x] = uint8_t(count.reads - 1);
		}
	const uint8_t* at = codes + triangles;
	uint32_t pending = 0; // varints to skip before the next aux byte or chunk start
	for (uint32_t first = 0, c = 0; first < triangles; first += chunk, ++c)
	{
		if (!skip_varints(at, aux, pending))
			return NVC_ERROR_CORRUPT;
		pending = 0;
		chunk_data[c] = uint64_t(at - stream);
		const uint32_t end = triangles - first < chunk ? triangles : first + chunk;
		for (uint32_t t = first; t < end; ++t)
		{
			const uint32_t code = codes[t];
			if (code < 0xfe)
				pending += varints[code];
			else
			{
				if (!skip_varints(at, aux, pending) || at == aux)
					return NVC_ERROR_CORRUPT;
				pending = varints_after[code & 1][*at++];
			}
		}
	}
	if (!skip_varints(at, aux, pending))
		return NVC_ERROR_CORRUPT;
	return at == aux ? version : NVC_ERROR_CORRUPT;
}

inline int decode_index_stream(const uint8_t* stream, size_t stream_size, uint32_t index_count, uint32_t* out)
{
	return decode_index_buffer(stream, stream_size, index_count, 4, out);
}

// The index-sequence codec into index_size (2 or 4) bytes per index
inline int decode_index_sequence(const uint8_t* stream, size_t stream_size, uint32_t index_count, uint32_t index_size, void* out)
{
	if (index_size != 2 && index_size != 4)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (stream_size < size_t(1) + index_count + 4) // at least one byte per index
		return NVC_ERROR_CORRUPT;
	if ((stream[0] & 0xf0) != 0xd0)
		return NVC_ERROR_CORRUPT;
	if ((stream[0] & 0x0f) > 1)
		return NVC_ERROR_UNSUPPORTED;
	// an index starts before the tail and may run into it (the tail is what makes a 5-byte varint readable); a stream is
	// well formed when the last index ends exactly at the tail
	const uint8_t* tail = stream + stream_size - 4;
	mhost::ByteReader r = { stream + 1, stream + stream_size };
	uint32_t last[2] = { 0, 0 };
	for (uint32_t i = 0; i < index_count; ++i)
	{
		uint32_t v;
		if (r.at >= tail || !mhost::read_varint(r, v))
			return NVC_ERROR_CORRUPT;
		const uint32_t base = v & 1u;
		v >>= 1;
		last[base] += (v >> 1) ^ (0u - (v & 1u));
		mhost::store_index(out, i, index_size, last[base]);
	}
	return r.at == tail ? NVC_OK : NVC_ERROR_CORRUPT;
}

// ---- vertex filters ---------------------------------------------------------------------------------------------------------
enum MeshoptFilter
{
	kFilterNone = NVC_MESHOPT_FILTER_NONE,
	kFilterOctahedral = NVC_MESHOPT_FILTER_OCTAHEDRAL,
	kFilterQuaternion = NVC_MESHOPT_FILTER_QUATERNION,
	kFilterExponential = NVC_MESHOPT_FILTER_EXPONENTIAL,
	kFilterColor = NVC_MESHOPT_FILTER_COLOR,
};

// the strides cgltf_validate accepts for a filter on an ATTRIBUTES view (a multiple of 4 up to 256, then the filter's own)
inline bool filter_stride_ok(int filter, uint32_t stride)
{
	if (stride == 0 || stride % 4 != 0 || stride > 256)
		return false;
	switch (filter)
	{
	case kFilterNone:
	case kFilterExponential: return true;
	case kFilterOctahedral:
	case kFilterColor: return stride == 4 || stride == 8;
	case kFilterQuaternion: return stride == 8;
	default: return false;
	}
}

namespace mhost
{

inline uint32_t float_bits(float f)
{
	uint32_t u;
	memcpy(&u, &f, 4);
	return u;
}

inline float bits_float(uint32_t u)
{
	float f;
	memcpy(&f, &u, 4);
	return f;
}

inline int32_t sign_extend(uint32_t v, int bits)
{
	return int32_t(v << (32 - bits)) >> (32 - bits);
}

// cvtps2dq: round to nearest even (the default rounding mode); NaN and values outside int32 give 0x80000000
inline uint32_t round_even(float f)
{
#ifdef NVC_FILTER_SSE
	return uint32_t(_mm_cvtss_si32(_mm_set_ss(f)));
#else
	if (!(f >= -2147483648.f && f < 2147483648.f))
		return 0x80000000u;
	return uint32_t(int32_t(nearbyintf(f)));
#endif
}

// rsqrtps / rcpps over four lanes: the approximations the CPU defines; exact elsewhere
inline void rsqrt4(float v[4])
{
#ifdef NVC_FILTER_SSE
	_mm_storeu_ps(v, _mm_rsqrt_ps(_mm_loadu_ps(v)));
#else
	for (int k = 0; k < 4; ++k)
		v[k] = 1.f / sqrtf(v[k]);
#endif
}

inline void rcp4(float v[4])
{
#ifdef NVC_FILTER_SSE
	_mm_storeu_ps(v, _mm_rcp_ps(_mm_loadu_ps(v)));
#else
	for (int k = 0; k < 4; ++k)
		v[k] = 1.f / v[k];
#endif
}

// x, y, z of an octahedral vector as the decoder reconstructs them before scaling; returns |v|^2
inline float unfold_octahedral(float& x, float& y, float& z, float zf)
{
	z = zf - (fabsf(x) + fabsf(y));
	const float t = z < 0.f ? z : 0.f;                               // minps(z, 0)
	x = x + bits_float(float_bits(t) ^ (float_bits(x) & 0x80000000u)); // t towards x's sign
	y = y + bits_float(float_bits(t) ^ (float_bits(y) & 0x80000000u));
	return x * x + (y * y + z * z);
}

// 4 elements of 4 bytes
inline void octahedral8(uint32_t* e)
{
	float x[4], y[4], z[4], s[4];
	for (int k = 0; k < 4; ++k)
	{
		x[k] = float(sign_extend(e[k], 8));
		y[k] = float(sign_extend(e[k] >> 8, 8));
		s[k] = unfold_octahedral(x[k], y[k], z[k], float(sign_extend(e[k] >> 16, 8)));
	}
	rsqrt4(s);
	for (int k = 0; k < 4; ++k)
	{
		const float scale = 127.f * s[k];
		e[k] = (e[k] & 0xff000000u) | (round_even(x[k] * scale) & 0xffu) | (round_even(y[k] * scale) & 0xffu) << 8 | (round_even(z[k] * scale) & 0xffu) << 16;
	}
}

// 4 elements of 4 x 16 bits
inline void octahedral16(uint16_t* e)
{
	for (int k = 0; k < 4; ++k)
	{
		uint16_t* v = e + 4 * k;
		float x = float(sign_extend(v[0], 16)), y = float(sign_extend(v[1], 16)), z;
		const float ll = unfold_octahedral(x, y, z, float(v[2] & 0x7fffu));
		const float scale = 32767.f / sqrtf(ll);
		v[0] = uint16_t(round_even(x * scale));
		v[1] = uint16_t(round_even(y * scale));
		v[2] = uint16_t(round_even(z * scale));
	}
}

inline void quaternion16(uint16_t* e)
{
	const float unit = 32767.f / sqrtf(2.f);
	for (int k = 0; k < 4; ++k)
	{
		uint16_t* v = e + 4 * k;
		const int32_t c = sign_extend(v[3], 16);
		const float s = float(c | 3);
		const float x = float(sign_extend(v[0], 16)), y = float(sign_extend(v[1], 16)), z = float(sign_extend(v[2], 16));
		const float ww = s * (s + s) - (x * x + (y * y + z * z));
		const float w = sqrtf(ww > 0.f ? ww : 0.f); // maxps(ww, 0)
		const float scale = unit / s;
		const uint64_t wxyz = uint64_t(round_even(w * scale) & 0xffffu) | uint64_t(round_even(x * scale) & 0xffffu) << 16 |
		    uint64_t(round_even(y * scale) & 0xffffu) << 32 | uint64_t(round_even(z * scale) & 0xffffu) << 48;
		const uint32_t rotate = uint32_t(c & 3) * 16u; // the dropped component moves to its place
		const uint64_t r = rotate ? (wxyz << rotate) | (wxyz >> (64u - rotate)) : wxyz;
		for (int j = 0; j < 4; ++j)
			v[j] = uint16_t(r >> (16 * j));
	}
}

inline void exponential(uint32_t* e)
{
	for (int k = 0; k < 4; ++k)
	{
		const uint32_t exponent = uint32_t(int32_t(e[k]) >> 24) + 127u;
		e[k] = float_bits(bits_float(exponent << 23) * float(sign_extend(e[k], 24)));
	}
}

// alpha's bit count from its highest set bit (all lower bits set), and alpha widened by one bit to the colour's count
inline uint32_t alpha_mask(uint32_t a, int bits)
{
	for (int shift = 1; shift < bits; shift *= 2)
		a |= a >> shift;
	return a;
}

inline void color8(uint32_t* e)
{
	int32_t y[4], co[4], cg[4];
	uint32_t a[4];
	float s[4];
	for (int k = 0; k < 4; ++k)
	{
		y[k] = int32_t(e[k] & 0xffu);
		co[k] = sign_extend(e[k] >> 8, 8);
		cg[k] = sign_extend(e[k] >> 16, 8);
		const uint32_t a8 = e[k] >> 24, mask = alpha_mask(a8, 8);
		a[k] = ((a8 << 1) & mask) | (a8 & 1u);
		s[k] = float(int32_t(mask));
	}
	rcp4(s);
	for (int k = 0; k < 4; ++k)
	{
		const float scale = 255.f * s[k];
		const uint32_t r = round_even(float(y[k] + (co[k] - cg[k])) * scale), g = round_even(float(y[k] + cg[k]) * scale);
		const uint32_t b = round_even(float(y[k] - (co[k] + cg[k])) * scale), al = round_even(float(int32_t(a[k])) * scale);
		e[k] = r | g << 8 | b << 16 | al << 24; // unmasked, as the SSE2 build combines them
	}
}

inline void color16(uint16_t* e)
{
	for (int k = 0; k < 4; ++k)
	{
		uint16_t* v = e + 4 * k;
		const int32_t y = v[0], co = sign_extend(v[1], 16), cg = sign_extend(v[2], 16);
		const uint32_t mask = alpha_mask(v[3], 16), a = ((uint32_t(v[3]) << 1) & mask) | (v[3] & 1u);
		const float scale = 65535.f / float(int32_t(mask));
		v[0] = uint16_t(round_even(float(y + (co - cg)) * scale));
		v[1] = uint16_t(round_even(float(y + cg) * scale));
		v[2] = uint16_t(round_even(float(y - (co + cg)) * scale));
		v[3] = uint16_t(round_even(float(int32_t(a)) * scale));
	}
}

// four `size`-byte elements at a time through a zeroed temporary; the last count % 4 leave the other lanes zero
template <typename Lane, typename Fn>
inline void filter_groups(uint8_t* data, size_t count, size_t size, Fn&& fn)
{
	for (size_t first = 0; first < count; first += 4)
	{
		const size_t n = count - first < 4 ? count - first : 4;
		Lane lanes[16] = {}; // room for 4 elements of up to 8 bytes
		memcpy(lanes, data + first * size, n * size);
		fn(lanes);
		memcpy(data + first * size, lanes, n * size);
	}
}

} // namespace mhost

// A filter applied in place to count elements of `stride` bytes; stride must pass filter_stride_ok
inline void decode_vertex_filter(int filter, uint8_t* data, size_t count, uint32_t stride)
{
	switch (filter)
	{
	case kFilterOctahedral:
		if (stride == 4)
			mhost::filter_groups<uint32_t>(data, count, 4, mhost::octahedral8);
		else
			mhost::filter_groups<uint16_t>(data, count, 8, mhost::octahedral16);
		break;
	case kFilterQuaternion: mhost::filter_groups<uint16_t>(data, count, 8, mhost::quaternion16); break;
	case kFilterExponential: mhost::filter_groups<uint32_t>(data, count * (stride / 4), 4, mhost::exponential); break;
	case kFilterColor:
		if (stride == 4)
			mhost::filter_groups<uint32_t>(data, count, 4, mhost::color8);
		else
			mhost::filter_groups<uint16_t>(data, count, 8, mhost::color16);
		break;
	default: break;
	}
}

} // namespace nvc
