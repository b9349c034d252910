// nvc_meshopt_encode.cpp — the index codec v1 (format in nvc_meshopt_decode.cpp) run backwards, for nvc_scene_cache_write.
// Host only: the codec is one sequential state machine, so the writer runs it on the host while the device encodes the
// vertex and meshlet streams.  The encoder keeps the decoder's own state (the vertex ring, the two edge rings, the next new
// vertex, the last explicit index) and, per triangle, picks the code the decoder turns back into it.  Where the format
// allows several codes, it makes the choices of saveSceneCache's encoder (meshopt_encodeIndexBuffer, version 1), so that
// the stream equals the reference's byte for byte:
//   - an edge of the triangle among the 15 newest edges, the newest one first; per edge slot the triangle's corners are
//     tried from (0, 1), then (1, 2), then (2, 0).  The third corner as: the vertex ring's slot when its newest copy is
//     in slots 2..13, else the next new vertex, else the last explicit index -/+ 1, else an explicit delta;
//   - otherwise a restart, the triangle rotated so that the next new vertex comes first when it is corner 1 or 2.  The
//     corners as: the next new vertex; for b and c also the ring slot when their newest copy is in slots 1..14; else
//     explicit.  (b, c) as one of the 14 first entries of the aux table when a is new, else as an explicit aux byte;
//   - a restart at 0, 1, 2 once the counter has moved resets it (explicit aux byte 0), and no vertex coded before the
//     reset is referred to through the ring afterwards.
#include "nvc_meshopt_format.h"

#include <string.h>

namespace nvc
{

namespace
{

// the aux table the reference's encoder writes at the end of every stream: (b, c) selector pairs of restarts
const uint8_t kAux[16] = { 0x00, 0x76, 0x87, 0x56, 0x67, 0x78, 0xa9, 0x86, 0x65, 0x89, 0x68, 0x98, 0x01, 0x69, 0x00, 0x00 };

// The newest slot n (1 = most recent) of the vertex ring that holds v, 0 when none does.  Only the `live` newest slots
// count; the reference's encoder sees the others as emptied (~0) after a reset, and so does this lookup.
uint32_t newest_slot(const icodec::Ring16& ring, uint32_t v, uint32_t live)
{
	for (uint32_t n = 1; n <= 16; ++n)
		if ((n <= live ? ring.back(n) : ~0u) == v)
			return n;
	return 0;
}

// a zigzag varint of index - last: 7 bits per byte, least significant first, the top bit set on all but the last byte
// (read_varint_delta reads it back)
uint8_t* put_delta(uint8_t* data, uint32_t index, uint32_t& last)
{
	const uint32_t d = index - last;
	uint32_t z = (d << 1) ^ (0u - (d >> 31));
	for (; z >= 128u; z >>= 7)
		*data++ = uint8_t(128u | (z & 127u));
	*data++ = uint8_t(z);
	last = index;
	return data;
}

} // namespace

size_t index_stream_bound(size_t index_count)
{
	return 1 + index_count / 3 * 17 + 16; // per triangle: code, aux byte, three 5-byte varints
}

size_t encode_index_stream(const uint32_t* indices, size_t index_count, uint8_t* stream)
{
	const size_t triangles = index_count / 3;
	stream[0] = 0xe1;
	uint8_t* codes = stream + 1;
	uint8_t* data = codes + triangles;
	icodec::Ring16 verts, edge_a, edge_b;
	// vertex ring slots the encoder may refer to: after a reset, none of the older ones
	uint32_t verts_live = 16;
	uint32_t next = 0, last = 0;
	auto push_edge = [&](uint32_t a, uint32_t b) {
		edge_a.put(a);
		edge_b.put(b);
	};

	for (size_t t = 0; t < triangles; ++t)
	{
		const uint32_t* tri = indices + 3 * t;
		// the newest edge slot e holding one of the triangle's directed edges, and the corner that edge starts at
		uint32_t e = 0, first = 0;
		for (uint32_t n = 1; n <= 15 && !e; ++n)
			for (uint32_t k = 0; k < 3 && !e; ++k)
				if (edge_a.back(n) == tri[k] && edge_b.back(n) == tri[(k + 1) % 3])
					e = n, first = k;
		if (e)
		{
			const uint32_t a = tri[first], b = tri[(first + 1) % 3], c = tri[(first + 2) % 3];
			const uint32_t n = newest_slot(verts, c, verts_live);
			uint32_t sel;
			if (n >= 2 && n <= 13)
				sel = n - 1; // direct slots 1..12 read back(sel + 1)
			else if (c == next)
				sel = 0, next++;
			else if (c == last - 1u)
				sel = 13, last = c;
			else if (c == last + 1u)
				sel = 14, last = c;
			else
			{
				sel = 15;
				data = put_delta(data, c, last);
			}
			codes[t] = uint8_t(((e - 1) << 4) | sel);
			verts.put(c, sel == 0 || sel >= 13);
			verts_live = sel == 0 || sel >= 13 ? (verts_live < 16 ? verts_live + 1 : 16) : verts_live;
			push_edge(c, b);
			push_edge(a, c);
			continue;
		}

		const uint32_t r = tri[1] == next ? 1u : tri[2] == next ? 2u : 0u;
		const uint32_t a = tri[r], b = tri[(r + 1) % 3], c = tri[(r + 2) % 3];
		const bool reset = a == 0 && b == 1 && c == 2 && next > 0;
		if (reset)
		{
			next = 0;
			verts_live = 0;
		}
		// ring slots are looked up before any corner of this triangle is pushed
		const uint32_t nb = newest_slot(verts, b, verts_live), nc = newest_slot(verts, c, verts_live);
		const uint32_t sel_a = a == next ? 0u : 15u;
		next += sel_a == 0;
		auto corner = [&](uint32_t v, uint32_t n) -> uint32_t {
			if (n >= 1 && n <= 14)
				return n;
			if (v == next)
			{
				next++;
				return 0;
			}
			return 15;
		};
		const uint32_t sel_b = corner(b, nb);
		const uint32_t sel_c = corner(c, nc);
		const uint8_t pair = uint8_t((sel_b << 4) | sel_c);
		const uint8_t* hit = reset || sel_a ? nullptr : static_cast<const uint8_t*>(memchr(kAux, pair, 14));
		if (hit)
			codes[t] = uint8_t(0xf0 | (hit - kAux));
		else
		{
			codes[t] = sel_a ? 0xff : 0xfe;
			*data++ = pair;
		}
		if (sel_a == 15)
			data = put_delta(data, a, last);
		if (sel_b == 15)
			data = put_delta(data, b, last);
		if (sel_c == 15)
			data = put_delta(data, c, last);
		verts.put(a);
		verts.put(b, sel_b == 0 || sel_b == 15);
		verts.put(c, sel_c == 0 || sel_c == 15);
		verts_live += 1 + (sel_b == 0 || sel_b == 15) + (sel_c == 0 || sel_c == 15);
		verts_live = verts_live < 16 ? verts_live : 16;
		push_edge(b, a);
		push_edge(c, b);
		push_edge(a, c);
	}
	memcpy(data, kAux, 16);
	return size_t(data + 16 - stream);
}

} // namespace nvc
