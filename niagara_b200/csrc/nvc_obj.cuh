// nvc_obj.cuh — OBJ import on the device (nvc_obj_load): loadMesh's loadObj (src/scene.cpp:117-168) over fast_obj's reader
// (extern/fast_obj/fast_obj.h), so that the Vertex[] is BIT-IDENTICAL to the reference's.
//
// Each line is a pure function of its bytes and of the v / vt / vn lines before it in its file; the only other link between
// lines is the reader's 64 KiB rule.  So the parse is data-parallel over lines, in four launch groups:
//   lines   per 4 KiB tile (256 threads x 16 bytes) its '\n' count, then their scan (nvc_scan.cuh's offsets_kernel).
//   count   each '\n' is written to its line slot; a full 64 KiB block without '\n' is flagged and the smallest flag of a file
//           is where the reader stops; one thread per line classifies it from its first bytes (a face line is walked to count
//           its records) and writes its counts (obj::Field), one row per field, which nvc_scan.cuh's device-wide scan
//           turns into prefixes, all rows in the same launches.  The scans run over all files at once: a file's values are
//           the prefix at its line minus the prefix at its first line.
//   parse   one thread per line writes its numbers, its index records and its face (window start, size, first corner); then
//           one thread per face checks the window loadObj reads (the running sum of face sizes, so orphan records shift it)
//           against the file's final counts.
//   expand  one thread per corner: its face by binary search over the faces' first corners, the fan position
//           (c0, c1, c2), (c0, c2, c3), ..., and one 16-byte store.
// A line's bytes are read through Line::at, which stands for '\n' at the line's end: no thread reads past its line.
// Numbers: fast_obj's parse_float restated in binary64 with every operation rounded on its own; an exponent's digits
// accumulate in a wrapping unsigned, and 20 or more multiplies by 0.0.  A NaN (inf / inf, inf * 0) is x86's default NaN,
// negative, so the float is 0xffc00000 whatever the device's NaN bits.  Indices: parse_int in 32-bit wrapping arithmetic.
#pragma once

#include "nvc_cook.cuh"
#include "nvc_internal.h"
#include "nvc_scan.cuh"

namespace nvc
{
namespace obj
{

constexpr uint32_t kThreads = 256;
constexpr uint32_t kNaN = 0xffc00000u;

// ---- one line's bytes -----------------------------------------------------------------------------------------------------

struct Line
{
	const uint8_t* text; // the file's first byte
	uint32_t end;        // the line's '\n' (or the file's end), file-relative

	__device__ __forceinline__ uint32_t at(uint32_t i) const { return i < end ? uint32_t(text[i]) : uint32_t('\n'); }
};

__device__ __forceinline__ bool is_space(uint32_t c) { return c == ' ' || c == '\t' || c == '\r'; }
__device__ __forceinline__ bool is_digit(uint32_t c) { return c - '0' < 10u; }

__device__ __forceinline__ uint32_t skip_space(const Line& l, uint32_t p)
{
	while (is_space(l.at(p)))
		++p;
	return p;
}

// fast_obj's POWER_10_POS / POWER_10_NEG[e], e < 20: the nearest doubles to 10^e and 10^-e
__device__ __forceinline__ double power_table(uint32_t e, bool negative)
{
	switch (e)
	{
	case 0: return 1.0e0;
	case 1: return negative ? 1.0e-1 : 1.0e1;
	case 2: return negative ? 1.0e-2 : 1.0e2;
	case 3: return negative ? 1.0e-3 : 1.0e3;
	case 4: return negative ? 1.0e-4 : 1.0e4;
	case 5: return negative ? 1.0e-5 : 1.0e5;
	case 6: return negative ? 1.0e-6 : 1.0e6;
	case 7: return negative ? 1.0e-7 : 1.0e7;
	case 8: return negative ? 1.0e-8 : 1.0e8;
	case 9: return negative ? 1.0e-9 : 1.0e9;
	case 10: return negative ? 1.0e-10 : 1.0e10;
	case 11: return negative ? 1.0e-11 : 1.0e11;
	case 12: return negative ? 1.0e-12 : 1.0e12;
	case 13: return negative ? 1.0e-13 : 1.0e13;
	case 14: return negative ? 1.0e-14 : 1.0e14;
	case 15: return negative ? 1.0e-15 : 1.0e15;
	case 16: return negative ? 1.0e-16 : 1.0e16;
	case 17: return negative ? 1.0e-17 : 1.0e17;
	case 18: return negative ? 1.0e-18 : 1.0e18;
	default: return negative ? 1.0e-19 : 1.0e19;
	}
}

// fast_obj.h:585-665 parse_float; returns the float's bits
__device__ __forceinline__ uint32_t parse_float(const Line& l, uint32_t& p)
{
	p = skip_space(l, p);
	double sign = 1.0;
	uint32_t c = l.at(p);
	if (c == '+')
		++p;
	else if (c == '-')
	{
		sign = -1.0;
		++p;
	}
	double num = 0.0;
	while (is_digit(c = l.at(p)))
	{
		num = __dadd_rn(__dmul_rn(10.0, num), double(c - '0'));
		++p;
	}
	if (c == '.')
		++p;
	double fra = 0.0, div = 1.0;
	while (is_digit(c = l.at(p)))
	{
		fra = __dadd_rn(__dmul_rn(10.0, fra), double(c - '0'));
		div = __dmul_rn(div, 10.0);
		++p;
	}
	num = __dadd_rn(num, __ddiv_rn(fra, div));
	if (c == 'e' || c == 'E')
	{
		++p;
		bool negative = false;
		c = l.at(p);
		if (c == '+')
			++p;
		else if (c == '-')
		{
			negative = true;
			++p;
		}
		uint32_t e = 0;
		while (is_digit(c = l.at(p)))
		{
			e = 10u * e + (c - '0');
			++p;
		}
		num = __dmul_rn(num, e >= 20u ? 0.0 : power_table(e, negative));
	}
	const double r = __dmul_rn(sign, num);
	return r != r ? kNaN : cook::float_bits(float(r));
}

// fast_obj.h:559-582 parse_int, in the 32-bit wrapping arithmetic of the reference's x86 build
__device__ __forceinline__ uint32_t parse_int(const Line& l, uint32_t& p)
{
	bool negative = false;
	if (l.at(p) == '-')
	{
		negative = true;
		++p;
	}
	uint32_t num = 0, c;
	while (is_digit(c = l.at(p)))
	{
		num = 10u * num + (c - '0');
		++p;
	}
	return negative ? 0u - num : num;
}

// fast_obj.h:769-788: an index against the array's size at this line (dummy element included)
__device__ __forceinline__ uint32_t resolve(uint32_t v, uint32_t size) { return int32_t(v) < 0 ? size - (0u - v) : v; }

// fast_obj.h:737-803 parse_face from just after "f ": emit(k, v, t, n) per index record pushed; returns the records pushed,
// and whether a face was pushed
template <typename Emit>
__device__ __forceinline__ uint32_t walk_face(const Line& l, uint32_t p, bool& face, const Emit& emit)
{
	p = skip_space(l, p);
	uint32_t count = 0;
	face = false;
	while (l.at(p) != '\n')
	{
		uint32_t t = 0, n = 0;
		const uint32_t v = parse_int(l, p);
		if (l.at(p) == '/')
		{
			++p;
			if (l.at(p) != '/')
				t = parse_int(l, p);
			if (l.at(p) == '/')
			{
				++p;
				n = parse_int(l, p);
			}
		}
		if (v == 0)
			return count;
		emit(count, v, t, n);
		++count;
		p = skip_space(l, p);
	}
	face = true;
	return count;
}

enum Kind : uint32_t
{
	kOther,
	kPosition,
	kTexcoord,
	kNormal,
	kFace
};

// fast_obj.h:1262-1304: the line's kind, and in `p` where its arguments start
__device__ __forceinline__ uint32_t classify(const Line& l, uint32_t start, uint32_t& p)
{
	p = skip_space(l, start);
	const uint32_t c0 = l.at(p), c1 = l.at(p + 1);
	p += 2;
	if (c0 == 'v')
		return c1 == ' ' || c1 == '\t' ? kPosition : c1 == 't' ? kTexcoord : c1 == 'n' ? kNormal : kOther;
	if (c0 == 'f')
		return c1 == ' ' || c1 == '\t' ? kFace : kOther;
	return kOther;
}

__device__ __forceinline__ uint32_t file_of_slot(const ObjArgs& a, uint32_t s)
{
	return scan::last_at_most(a.file_count, s, [&](uint32_t f) { return a.state[f].first_line; });
}

__device__ __forceinline__ Line line_of(const ObjArgs& a, uint32_t f, uint32_t s, uint32_t& start)
{
	start = s == a.state[f].first_line ? 0u : a.line_end[s - 1] + 1u;
	return Line{ a.text + a.files[f].data, a.line_end[s] };
}

__device__ __forceinline__ unsigned long long prefix(const ObjArgs& a, uint32_t field, uint32_t s)
{
	return a.prefix[uint64_t(field) * (uint64_t(a.line_slots) + 1) + s];
}

// ---- lines ----------------------------------------------------------------------------------------------------------------

// thread x of tile t: its 16 bytes (fewer at the file's end) and how many are '\n'
struct TileBytes
{
	uint8_t b[16];
	uint32_t n;     // bytes present
	uint32_t pos;   // file-relative position of b[0]
	uint32_t file;
};

__device__ __forceinline__ TileBytes tile_bytes(const ObjArgs& a, uint32_t t)
{
	TileBytes r;
	r.file = scan::last_at_most(a.file_count, t, [&](uint32_t f) { return a.files[f].tile_base; });
	const File& f = a.files[r.file];
	r.pos = (t - f.tile_base) * kTileBytes + threadIdx.x * 16u;
	r.n = r.pos < f.size ? min(16u, f.size - r.pos) : 0u;
	const uint8_t* src = a.text + f.data + r.pos;
	if (r.n == 16 && (reinterpret_cast<uintptr_t>(src) & 15u) == 0) // always aligned in device memory (cudaMalloc)
	{
		const uint4 w = *reinterpret_cast<const uint4*>(src);
		memcpy(r.b, &w, 16);
	}
	else
		for (uint32_t k = 0; k < 16; ++k)
			r.b[k] = k < r.n ? src[k] : 0;
	return r;
}

__device__ __forceinline__ uint32_t newlines(const TileBytes& r)
{
	uint32_t c = 0;
	for (uint32_t k = 0; k < 16; ++k)
		c += k < r.n && r.b[k] == '\n';
	return c;
}

__global__ void __launch_bounds__(kThreads) obj_tile_count_kernel(const ObjArgs a)
{
	__shared__ uint32_t s_warp[kThreads / 32];
	const uint32_t total = scan::block_sum<kThreads>(newlines(tile_bytes(a, blockIdx.x)), s_warp);
	if (threadIdx.x == 0)
		a.tile_lines[blockIdx.x] = total;
}

// ---- count ----------------------------------------------------------------------------------------------------------------

// line_end[tile_offsets[t] + file + k] = the k-th '\n' of tile t
__global__ void __launch_bounds__(kThreads) obj_line_end_kernel(const ObjArgs a)
{
	__shared__ uint32_t s_warp[kThreads / 32];
	const TileBytes r = tile_bytes(a, blockIdx.x);
	uint32_t total;
	uint64_t slot = a.tile_offsets[blockIdx.x] + r.file + scan::block_exclusive<kThreads>(newlines(r), s_warp, total);
	for (uint32_t k = 0; k < 16; ++k)
		if (k < r.n && r.b[k] == '\n')
			a.line_end[slot++] = r.pos + k;
}

// one thread per tile that starts a 64 KiB block: a full block without '\n' is a cut candidate of its file
__global__ void __launch_bounds__(kThreads) obj_cut_kernel(const ObjArgs a)
{
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	if (t >= a.tile_count)
		return;
	const uint32_t f = scan::last_at_most(a.file_count, t, [&](uint32_t g) { return a.files[g].tile_base; });
	const uint32_t j = t - a.files[f].tile_base;
	if (j % kTilesPerBlock != 0 || uint64_t(j + kTilesPerBlock) * kTileBytes > a.files[f].size)
		return;
	if (a.tile_offsets[t + kTilesPerBlock] == a.tile_offsets[t])
		atomicMin(&a.state[f].cut, j / kTilesPerBlock);
}

// one thread per file: its line slots and the lines the reader parses (fast_obj.h:1501-1552)
__global__ void __launch_bounds__(kThreads) obj_file_kernel(const ObjArgs a)
{
	const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
	if (f >= a.file_count)
		return;
	const File& file = a.files[f];
	FileState& s = a.state[f];
	const unsigned long long base = a.tile_offsets[file.tile_base];
	const uint32_t total = uint32_t(a.tile_offsets[a.files[f + 1].tile_base] - base);
	s.first_line = uint32_t(base) + f;
	s.flags = 0;
	if (s.cut != ~0u)
		s.line_count = uint32_t(a.tile_offsets[file.tile_base + s.cut * kTilesPerBlock] - base);
	else
	{
		// the last block gets a '\n' when it lacks one: a final line without '\n' ends at the file's end
		const bool open = file.size && a.text[file.data + file.size - 1] != '\n';
		s.line_count = total + (open ? 1u : 0u);
		a.line_end[s.first_line + total] = file.size;
	}
}

__global__ void __launch_bounds__(kThreads) obj_classify_kernel(const ObjArgs a)
{
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s >= a.line_slots)
		return;
	const uint64_t L = a.line_slots;
	uint32_t c[kFields] = {};
	const uint32_t f = file_of_slot(a, s);
	if (s - a.state[f].first_line < a.state[f].line_count)
	{
		uint32_t start, p;
		const Line l = line_of(a, f, s, start);
		const uint32_t kind = classify(l, start, p);
		c[kPositions] = kind == kPosition;
		c[kTexcoords] = kind == kTexcoord;
		c[kNormals] = kind == kNormal;
		if (kind == kFace)
		{
			bool face;
			const uint32_t n = walk_face(l, p, face, [](uint32_t, uint32_t, uint32_t, uint32_t) {});
			c[kRecords] = n;
			c[kFaces] = face;
			c[kFaceIndices] = face ? n : 0u;
			c[kCorners] = face && n >= 3 ? 3u * (n - 2u) : 0u;
			if (face && n < 3)
				atomicOr(&a.state[f].flags, kBadFace);
		}
	}
	for (uint32_t k = 0; k < kFields; ++k)
		a.counts[k * L + s] = c[k];
}

// one thread per file: its final counts, its arrays' bases, its info
__global__ void __launch_bounds__(kThreads) obj_info_kernel(const ObjArgs a)
{
	const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
	if (f >= a.file_count)
		return;
	FileState& s = a.state[f];
	const uint32_t lo = s.first_line, hi = f + 1 < a.file_count ? a.state[f + 1].first_line : a.line_slots;
	auto total = [&](uint32_t k) { return prefix(a, k, hi) - prefix(a, k, lo); };
	s.positions = uint32_t(total(kPositions));
	s.texcoords = uint32_t(total(kTexcoords));
	s.normals = uint32_t(total(kNormals));
	s.position_base = prefix(a, kPositions, lo) + f;
	s.texcoord_base = prefix(a, kTexcoords, lo) + f;
	s.normal_base = prefix(a, kNormals, lo) + f;
	NvcObjInfo& info = a.infos[f];
	info.bytes_parsed = s.cut == ~0u ? a.files[f].size : (s.line_count ? a.line_end[lo + s.line_count - 1] + 1ull : 0ull);
	info.position_count = s.positions;
	info.texcoord_count = s.texcoords;
	info.normal_count = s.normals;
	info.face_count = uint32_t(total(kFaces));
	info.index_count = total(kRecords);
	info.corner_offset = prefix(a, kCorners, lo);
	info.corner_count = total(kCorners);
}

// ---- parse ----------------------------------------------------------------------------------------------------------------

// each file's dummy elements (fast_obj.h:1464-1474): position (0, 0, 0), texcoord (0, 0), normal (0, 0, 1)
__global__ void __launch_bounds__(kThreads) obj_dummy_kernel(const ObjArgs a)
{
	const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
	if (f >= a.file_count)
		return;
	const FileState& s = a.state[f];
	for (uint32_t k = 0; k < 3; ++k)
		a.positions[3 * s.position_base + k] = 0.0f;
	a.texcoords[2 * s.texcoord_base + 0] = 0.0f;
	a.texcoords[2 * s.texcoord_base + 1] = 0.0f;
	a.normals[3 * s.normal_base + 0] = 0.0f;
	a.normals[3 * s.normal_base + 1] = 0.0f;
	a.normals[3 * s.normal_base + 2] = 1.0f;
}

__global__ void __launch_bounds__(kThreads) obj_parse_kernel(const ObjArgs a)
{
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s >= a.line_slots)
		return;
	const uint32_t f = file_of_slot(a, s);
	const FileState& st = a.state[f];
	if (s - st.first_line >= st.line_count)
		return;
	uint32_t start, p;
	const Line l = line_of(a, f, s, start);
	const uint32_t kind = classify(l, start, p);
	if (kind == kPosition || kind == kNormal)
	{
		// the file's element index is its prefix within the file + 1 (after the dummy) = the global prefix + the file's index + 1
		float* dst = (kind == kPosition ? a.positions : a.normals) + 3 * (prefix(a, kind == kPosition ? kPositions : kNormals, s) + f + 1);
		for (uint32_t k = 0; k < 3; ++k)
			dst[k] = cook::bits_float(parse_float(l, p));
	}
	else if (kind == kTexcoord)
	{
		float* dst = a.texcoords + 2 * (prefix(a, kTexcoords, s) + f + 1);
		for (uint32_t k = 0; k < 2; ++k)
			dst[k] = cook::bits_float(parse_float(l, p));
	}
	else if (kind == kFace)
	{
		const uint32_t lo = st.first_line;
		// the arrays' sizes at this line, dummy included (fast_obj.h:770-784)
		const uint32_t np = uint32_t(prefix(a, kPositions, s) - prefix(a, kPositions, lo)) + 1;
		const uint32_t nt = uint32_t(prefix(a, kTexcoords, s) - prefix(a, kTexcoords, lo)) + 1;
		const uint32_t nn = uint32_t(prefix(a, kNormals, s) - prefix(a, kNormals, lo)) + 1;
		Record* dst = a.records + prefix(a, kRecords, s);
		bool face;
		const uint32_t n = walk_face(l, p, face, [&](uint32_t k, uint32_t v, uint32_t t, uint32_t nv) {
			dst[k] = Record{ resolve(v, np), resolve(t, nt), resolve(nv, nn) };
		});
		if (face)
		{
			Face r;
			r.window = uint32_t(prefix(a, kRecords, lo) + (prefix(a, kFaceIndices, s) - prefix(a, kFaceIndices, lo)));
			r.count = n;
			r.file = f;
			r.pad = 0;
			r.corner = prefix(a, kCorners, s);
			a.faces[prefix(a, kFaces, s)] = r;
		}
	}
}

// one thread per face: the window loadObj reads, against the file's final counts
__global__ void __launch_bounds__(kThreads) obj_check_kernel(const ObjArgs a)
{
	const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
	if (i >= a.face_count)
		return;
	const Face face = a.faces[i];
	const FileState& s = a.state[face.file];
	bool bad = false;
	for (uint32_t k = 0; k < face.count; ++k)
	{
		const Record r = a.records[face.window + k];
		bad = bad || r.p > s.positions || r.t > s.texcoords || r.n > s.normals;
	}
	if (bad)
		atomicOr(&a.state[face.file].flags, kBadIndex);
}

// ---- expand ---------------------------------------------------------------------------------------------------------------

// scene.cpp:133-161: one thread per corner
__global__ void __launch_bounds__(kThreads) obj_expand_kernel(const ObjArgs a)
{
	const uint64_t c = uint64_t(blockIdx.x) * kThreads + threadIdx.x;
	if (c >= a.corner_count)
		return;
	const uint32_t i = scan::last_at_most(a.face_count, c, [&](uint32_t k) { return a.faces[k].corner; });
	const Face face = a.faces[i];
	const uint32_t j = uint32_t(c - face.corner), r = j % 3;
	const uint32_t fan = r == 0 ? 0 : j / 3 + r; // (c0, c(k+1), c(k+2)) for triangle k
	const Record rec = a.records[face.window + fan];
	const FileState& s = a.state[face.file];
	const float* pos = a.positions + 3 * (s.position_base + rec.p);
	const float* nrm = a.normals + 3 * (s.normal_base + rec.n);
	const float* tex = a.texcoords + 2 * (s.texcoord_base + rec.t);
	uint4 w;
	w.x = uint32_t(cook::quantize_half(pos[0])) | uint32_t(cook::quantize_half(pos[1])) << 16;
	w.y = uint32_t(cook::quantize_half(pos[2]));
	w.z = uint32_t(cook::quantize_snorm(nrm[0], 10) + 511) | uint32_t(cook::quantize_snorm(nrm[1], 10) + 511) << 10 |
	      uint32_t(cook::quantize_snorm(nrm[2], 10) + 511) << 20;
	w.w = uint32_t(cook::quantize_half(tex[0])) | uint32_t(cook::quantize_half(tex[1])) << 16;
	reinterpret_cast<uint4*>(a.vertices)[c] = w;
}

} // namespace obj
} // namespace nvc
