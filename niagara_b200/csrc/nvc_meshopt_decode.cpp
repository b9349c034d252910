// nvc_meshopt_decode.cpp — decoders for the two remaining meshopt streams of a compressed scene cache (row N2):
// the vertex codec (scenecache.cpp:64-72,244-248: vertices and the RT position stream) and the index codec
// (:74-82,250-254).  Host only.  Both are lossless, so the check is simple: decoding the compressed cache the
// reference wrote must give the bytes of the uncompressed cache it wrote (tests/test_scene_cache.py).
//
// Formats (meshoptimizer v1.0, extern/meshoptimizer/src/vertexcodec.cpp, indexcodec.cpp — restated, not copied):
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
#include "../../include/niagara_cull.h"
#include "nvc_meshopt_format.h"

#include <string.h>

namespace nvc
{

namespace
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
bool walk_plane(ByteReader& r, int control, int version, uint32_t count, Group&& group)
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

bool read_plane(ByteReader& r, int control, int version, uint32_t count, uint8_t* out /* room for count rounded up to 16 */)
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

int open_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t stride, VertexStream& out)
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

} // namespace

// 0 ok, negative NvcStatus otherwise
int decode_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t vertex_count, uint32_t stride, uint8_t* out)
{
	VertexStream vs;
	int status = open_vertex_stream(stream, stream_size, stride, vs);
	if (status != NVC_OK)
		return status;
	const int version = vs.version;
	const uint8_t* channels = vs.channels;
	uint8_t previous[256];
	memcpy(previous, vs.baseline, stride);
	ByteReader& r = vs.blocks;
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
				if (!read_plane(r, int((ctrl >> (j * 2)) & 3u), version, count, planes[j]))
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
int walk_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t vertex_count, uint32_t stride, uint32_t* block_start, uint16_t* plane_offset,
    VertexStreamTail* tail)
{
	if (stride > 16)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (stream_size > 0xffffffffull)
		return NVC_ERROR_UNSUPPORTED; // block starts are 32-bit offsets
	VertexStream vs;
	int status = open_vertex_stream(stream, stream_size, stride, vs);
	if (status != NVC_OK)
		return status;
	tail->version = vs.version;
	tail->baseline = vs.baseline;
	tail->channels = vs.channels;
	ByteReader& r = vs.blocks;
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
			if (!walk_plane(r, int(ctrl), vs.version, count, nothing))
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

namespace
{

bool read_varint_delta(ByteReader& r, uint32_t& last)
{
	uint32_t value = 0;
	for (int i = 0; i < 5; ++i)
	{
		const uint8_t* b;
		if (!r.take(1, b))
			return false;
		value |= uint32_t(*b & 127u) << (7 * i);
		if (*b < 128)
			break;
	}
	last += (value >> 1) ^ (0u - (value & 1u));
	return true;
}

} // namespace

int decode_index_stream(const uint8_t* stream, size_t stream_size, uint32_t index_count, uint32_t* out)
{
	if (index_count % 3 != 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	const uint32_t triangles = index_count / 3;
	if (stream_size < size_t(1) + triangles + 16)
		return NVC_ERROR_CORRUPT;
	if ((stream[0] & 0xf0) != 0xe0)
		return NVC_ERROR_CORRUPT;
	const int version = stream[0] & 0x0f;
	if (version > 1)
		return NVC_ERROR_UNSUPPORTED;
	const uint32_t direct_slots = version >= 1 ? 13u : 15u;

	const uint8_t* codes = stream + 1;
	const uint8_t* aux = stream + stream_size - 16;
	ByteReader r = { codes + triangles, aux };

	icodec::Ring16 verts, edge_a, edge_b;
	auto push_edge = [&](uint32_t a, uint32_t b) {
		edge_a.put(a);
		edge_b.put(b);
	};
	uint32_t next = 0, last = 0;

	for (uint32_t t = 0; t < triangles; ++t)
	{
		const uint32_t code = codes[t];
		uint32_t a, b, c;
		if (code < 0xf0)
		{
			uint32_t e = (code >> 4) + 1u;
			a = edge_a.back(e);
			b = edge_b.back(e);
			uint32_t sel = code & 15u;
			if (sel < direct_slots)
			{
				c = sel == 0 ? next : verts.back(sel + 1u);
				next += sel == 0 ? 1u : 0u;
				verts.put(c, sel == 0);
			}
			else
			{
				if (sel == 15u)
				{
					if (!read_varint_delta(r, last))
						return NVC_ERROR_CORRUPT;
				}
				else
					last += sel == 13u ? 0xffffffffu : 1u; // 13 -> -1, 14 -> +1
				c = last;
				verts.put(c);
			}
			push_edge(c, b);
			push_edge(a, c);
		}
		else
		{
			uint32_t sel_a = 0, sel_b, sel_c;
			if (code < 0xfe)
			{
				uint32_t x = aux[code & 15u];
				sel_b = x >> 4;
				sel_c = x & 15u;
			}
			else
			{
				const uint8_t* x;
				if (!r.take(1, x))
					return NVC_ERROR_CORRUPT;
				sel_a = code == 0xfe ? 0u : 15u;
				sel_b = *x >> 4;
				sel_c = *x & 15u;
				if (*x == 0)
					next = 0;
			}
			// FIFO lookups use the ring as it is BEFORE this triangle's vertices are pushed
			a = sel_a == 0 ? next++ : 0u;
			b = sel_b == 0 ? next++ : verts.back(sel_b);
			c = sel_c == 0 ? next++ : verts.back(sel_c);
			if (sel_a == 15u)
			{
				if (!read_varint_delta(r, last))
					return NVC_ERROR_CORRUPT;
				a = last;
			}
			if (sel_b == 15u)
			{
				if (!read_varint_delta(r, last))
					return NVC_ERROR_CORRUPT;
				b = last;
			}
			if (sel_c == 15u)
			{
				if (!read_varint_delta(r, last))
					return NVC_ERROR_CORRUPT;
				c = last;
			}
			verts.put(a);
			verts.put(b, sel_b == 0 || sel_b == 15u);
			verts.put(c, sel_c == 0 || sel_c == 15u);
			push_edge(b, a);
			push_edge(c, b);
			push_edge(a, c);
		}
		out[size_t(t) * 3 + 0] = a;
		out[size_t(t) * 3 + 1] = b;
		out[size_t(t) * 3 + 2] = c;
	}
	return r.at == r.end ? NVC_OK : NVC_ERROR_CORRUPT;
}

} // namespace nvc
