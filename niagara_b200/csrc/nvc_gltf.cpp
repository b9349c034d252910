// nvc_gltf.cpp — glTF 2.0 scene import for the visibility path (row N3 of SURVEY §8(f)): what loadScene
// (src/scene.cpp:473-853) produces for the frame loop — MeshDraw[] (world transform of every mesh node decomposed into
// position / uniform scale / orientation, meshIndex per triangle primitive, materialIndex, postPass from the material's
// alpha mode / transmission), Animation[] + Keyframe[] (LINEAR TRS samplers baked per key through the node hierarchy), the
// camera, the sun direction — plus, per primitive, the quantised Vertex[] / index arrays loadVertices builds (the geometry
// cooker that turns those into Mesh / Meshlet tables stays out of scope; the scene cache carries its output).
//
// Written from the glTF 2.0 specification; no third-party parser.  Where results must equal the reference's bit for bit
// the arithmetic follows what the reference executes, cited per function: numbers are parsed as double and narrowed to
// float (cgltf: CGLTF_ATOF = atof), node matrices are composed in binary32 in the order of cgltf_node_transform_local /
// _world (extern/cgltf/cgltf.h:2137-2216), decomposeTransform is scene.cpp:295-340.  Host code, strict IEEE
// (-ffp-contract=off).  Supported: .gltf with data: URIs or external buffers, .glb; dense accessors of every component
// type; TRS or matrix nodes; KHR_materials_transmission (presence), KHR_lights_punctual (directional -> sun, point -> light
// slots for animation targets), EXT_meshopt_compression / KHR_meshopt_compression (below).  Not supported
// (NVC_ERROR_UNSUPPORTED): sparse accessors.
//
// Meshopt compression, as loadScene's decompressMeshopt (scene.cpp:405-470) runs it after cgltf_validate: every buffer view
// with the extension (buffer, byteOffset, byteLength, byteStride, count, mode, filter; cgltf.h:5045-5130, both extension
// names parse alike) is checked against cgltf_validate's rules (cgltf.h:1640-1667) and decoded at import, whether a used
// primitive reads it or not, with the decoders of nvc_meshopt_host.h (inline, so that this file links on its own).  The
// decoded bytes replace the view's contents for every accessor.  A buffer without data is accepted when it declares itself a
// meshopt fallback buffer ("fallback": true: gltfpack writes the compressed views' uncompressed size there and no bytes);
// an uncompressed view into it is refused.
#include "../../include/niagara_cull.h"
#include "nvc_meshopt_host.h"

#include <ctype.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <new>
#include <string>
#include <vector>

namespace
{

// ---- a small JSON document ------------------------------------------------------------------------------------------------
struct Json
{
	enum Type
	{
		Null,
		Bool,
		Number,
		String,
		Array,
		Object
	} type = Null;
	bool b = false;
	double num = 0;
	std::string str;
	std::vector<Json> items;                           // Array
	std::vector<std::pair<std::string, Json>> members; // Object (insertion order)

	const Json* get(const char* key) const
	{
		if (type != Object)
			return nullptr;
		for (const auto& m : members)
			if (m.first == key)
				return &m.second;
		return nullptr;
	}
	size_t size() const { return type == Array ? items.size() : 0; }
	const Json& at(size_t i) const { return items[i]; }
	bool is_number() const { return type == Number; }
};

struct JsonParser
{
	const char* p;
	const char* end;
	bool ok = true;
	int depth = 0;

	void ws()
	{
		while (p < end && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r'))
			++p;
	}
	bool lit(const char* s)
	{
		size_t n = strlen(s);
		if (size_t(end - p) >= n && memcmp(p, s, n) == 0)
		{
			p += n;
			return true;
		}
		return false;
	}
	static void utf8(std::string& out, uint32_t c)
	{
		if (c < 0x80)
			out.push_back(char(c));
		else if (c < 0x800)
		{
			out.push_back(char(0xc0 | (c >> 6)));
			out.push_back(char(0x80 | (c & 0x3f)));
		}
		else if (c < 0x10000)
		{
			out.push_back(char(0xe0 | (c >> 12)));
			out.push_back(char(0x80 | ((c >> 6) & 0x3f)));
			out.push_back(char(0x80 | (c & 0x3f)));
		}
		else
		{
			out.push_back(char(0xf0 | (c >> 18)));
			out.push_back(char(0x80 | ((c >> 12) & 0x3f)));
			out.push_back(char(0x80 | ((c >> 6) & 0x3f)));
			out.push_back(char(0x80 | (c & 0x3f)));
		}
	}
	bool hex4(uint32_t& v)
	{
		if (end - p < 4)
			return false;
		v = 0;
		for (int i = 0; i < 4; ++i)
		{
			char c = *p++;
			v <<= 4;
			if (c >= '0' && c <= '9')
				v |= uint32_t(c - '0');
			else if (c >= 'a' && c <= 'f')
				v |= uint32_t(c - 'a' + 10);
			else if (c >= 'A' && c <= 'F')
				v |= uint32_t(c - 'A' + 10);
			else
				return false;
		}
		return true;
	}
	bool string(std::string& out)
	{
		if (p >= end || *p != '"')
			return false;
		++p;
		while (p < end && *p != '"')
		{
			char c = *p++;
			if (c != '\\')
			{
				out.push_back(c);
				continue;
			}
			if (p >= end)
				return false;
			char e = *p++;
			switch (e)
			{
			case '"': out.push_back('"'); break;
			case '\\': out.push_back('\\'); break;
			case '/': out.push_back('/'); break;
			case 'b': out.push_back('\b'); break;
			case 'f': out.push_back('\f'); break;
			case 'n': out.push_back('\n'); break;
			case 'r': out.push_back('\r'); break;
			case 't': out.push_back('\t'); break;
			case 'u': {
				uint32_t v;
				if (!hex4(v))
					return false;
				if (v >= 0xd800 && v < 0xdc00 && end - p >= 6 && p[0] == '\\' && p[1] == 'u')
				{
					p += 2;
					uint32_t lo;
					if (!hex4(lo))
						return false;
					v = 0x10000 + ((v - 0xd800) << 10) + (lo - 0xdc00);
				}
				utf8(out, v);
				break;
			}
			default: return false;
			}
		}
		if (p >= end)
			return false;
		++p;
		return true;
	}
	Json value()
	{
		Json j;
		if (++depth > 64)
		{
			ok = false;
			return j;
		}
		ws();
		if (p >= end)
			ok = false;
		else if (*p == '{')
		{
			++p;
			j.type = Json::Object;
			ws();
			if (p < end && *p == '}')
				++p;
			else
				for (;;)
				{
					ws();
					std::string key;
					if (!string(key))
					{
						ok = false;
						break;
					}
					ws();
					if (p >= end || *p != ':')
					{
						ok = false;
						break;
					}
					++p;
					Json v = value();
					if (!ok)
						break;
					j.members.emplace_back(std::move(key), std::move(v));
					ws();
					if (p < end && *p == ',')
					{
						++p;
						continue;
					}
					if (p < end && *p == '}')
					{
						++p;
						break;
					}
					ok = false;
					break;
				}
		}
		else if (*p == '[')
		{
			++p;
			j.type = Json::Array;
			ws();
			if (p < end && *p == ']')
				++p;
			else
				for (;;)
				{
					Json v = value();
					if (!ok)
						break;
					j.items.push_back(std::move(v));
					ws();
					if (p < end && *p == ',')
					{
						++p;
						continue;
					}
					if (p < end && *p == ']')
					{
						++p;
						break;
					}
					ok = false;
					break;
				}
		}
		else if (*p == '"')
		{
			j.type = Json::String;
			ok = string(j.str);
		}
		else if (lit("true"))
		{
			j.type = Json::Bool;
			j.b = true;
		}
		else if (lit("false"))
			j.type = Json::Bool;
		else if (lit("null"))
			j.type = Json::Null;
		else
		{
			// number: the reference's parser hands the token to atof (CGLTF_ATOF), i.e. strtod
			const char* s = p;
			while (p < end && (*p == '-' || *p == '+' || *p == '.' || *p == 'e' || *p == 'E' || (*p >= '0' && *p <= '9')))
				++p;
			if (p == s)
				ok = false;
			else
			{
				std::string tok(s, p);
				char* stop = nullptr;
				j.num = strtod(tok.c_str(), &stop);
				j.type = Json::Number;
				if (!stop || *stop)
					ok = false;
			}
		}
		--depth;
		return j;
	}
};

float num_f(const Json* j, float def)
{
	return j && j->is_number() ? float(j->num) : def;
}
long long num_i(const Json* j, long long def)
{
	return j && j->is_number() ? (long long)(j->num) : def;
}

// ---- glTF objects ---------------------------------------------------------------------------------------------------------
struct BufferView
{
	size_t buffer = 0, offset = 0, length = 0, stride = 0;
};
struct Accessor
{
	long long view = -1;
	size_t offset = 0, count = 0;
	int component = 0; // 5120 s8, 5121 u8, 5122 s16, 5123 u16, 5125 u32, 5126 f32
	int components = 0;
	bool normalized = false;
};
struct Primitive
{
	long long position = -1, normal = -1, tangent = -1, texcoord = -1, indices = -1, material = -1;
	int mode = 4;
};
struct Node
{
	float translation[3] = { 0, 0, 0 }, rotation[4] = { 0, 0, 0, 1 }, scale[3] = { 1, 1, 1 }, matrix[16];
	bool has_matrix = false;
	long long mesh = -1, camera = -1, light = -1, parent = -1;
};
struct Sampler
{
	long long input = -1, output = -1;
	bool linear = true;
};

} // namespace

struct NvcGltfScene
{
	std::vector<std::vector<uint8_t>> buffers; // the file's buffers, then one per decoded meshopt view
	std::vector<uint64_t> buffer_length;       // byteLength as declared (what cgltf_validate checks views against)
	std::vector<bool> buffer_fallback;         // a meshopt fallback buffer: no data
	std::vector<BufferView> views;
	std::vector<Accessor> accessors;
	std::vector<std::vector<Primitive>> meshes;
	std::vector<Node> nodes;
	std::vector<uint8_t> material_post_pass; // 0 opaque, 1 alpha (mask / blend), 2 transmission
	std::vector<float> camera_yfov;
	std::vector<int> light_type; // 0 other, 1 directional, 2 point
	// results
	NvcGltfInfo info;
	std::vector<NvcMeshDraw> draws;
	std::vector<NvcAnimation> animations;
	std::vector<NvcKeyframe> keyframes;
	std::vector<float> mesh_scale; // per glTF mesh: max |cbrt(det(world))| over its nodes (scene.cpp:503-519)
	struct Prim
	{
		uint32_t mesh, index_in_mesh;
		const Primitive* p;
	};
	std::vector<Prim> primitives; // triangle primitives with indices, in meshIndex order
	std::string error;
};

namespace
{

int fail(NvcGltfScene* s, int code, const std::string& what)
{
	s->error = what;
	return code;
}

int b64(char c)
{
	if (c >= 'A' && c <= 'Z')
		return c - 'A';
	if (c >= 'a' && c <= 'z')
		return c - 'a' + 26;
	if (c >= '0' && c <= '9')
		return c - '0' + 52;
	if (c == '+' || c == '-')
		return 62;
	if (c == '/' || c == '_')
		return 63;
	return -1;
}

bool decode_base64(const char* s, size_t n, std::vector<uint8_t>& out)
{
	uint32_t acc = 0;
	int bits = 0;
	for (size_t i = 0; i < n; ++i)
	{
		if (s[i] == '=')
			break;
		int v = b64(s[i]);
		if (v < 0)
			return false;
		acc = (acc << 6) | uint32_t(v);
		bits += 6;
		if (bits >= 8)
		{
			bits -= 8;
			out.push_back(uint8_t(acc >> bits));
		}
	}
	return true;
}

bool read_file(const std::string& path, std::vector<uint8_t>& out)
{
	FILE* f = fopen(path.c_str(), "rb");
	if (!f)
		return false;
	fseek(f, 0, SEEK_END);
	long n = ftell(f);
	fseek(f, 0, SEEK_SET);
	out.resize(n > 0 ? size_t(n) : 0);
	bool ok = n >= 0 && fread(out.data(), 1, out.size(), f) == out.size();
	fclose(f);
	return ok;
}

int component_size(int c)
{
	switch (c)
	{
	case 5120:
	case 5121: return 1;
	case 5122:
	case 5123: return 2;
	case 5125:
	case 5126: return 4;
	default: return 0;
	}
}

// element `index` of a dense accessor; nullptr when it does not lie inside its buffer
const uint8_t* element(const NvcGltfScene& s, const Accessor& a, size_t index, size_t* out_stride = nullptr)
{
	if (a.view < 0 || size_t(a.view) >= s.views.size())
		return nullptr;
	const BufferView& v = s.views[size_t(a.view)];
	if (v.buffer >= s.buffers.size())
		return nullptr;
	const size_t esize = size_t(component_size(a.component)) * size_t(a.components);
	const size_t stride = v.stride ? v.stride : esize;
	if (out_stride)
		*out_stride = stride;
	const std::vector<uint8_t>& b = s.buffers[v.buffer];
	const uint64_t at = uint64_t(v.offset) + a.offset + uint64_t(index) * stride;
	if (esize == 0 || at + esize > b.size() || a.offset + uint64_t(index) * stride + esize > v.length)
		return nullptr;
	return b.data() + at;
}

// cgltf_component_read_float (cgltf.h:2251-2277): floats verbatim, normalized integers / (float)max, others (float)int
float component_float(const uint8_t* in, int component, bool normalized)
{
	switch (component)
	{
	case 5126: {
		float f;
		memcpy(&f, in, 4);
		return f;
	}
	case 5120: {
		int8_t v;
		memcpy(&v, in, 1);
		return normalized ? v / 127.0f : float(v);
	}
	case 5121: return normalized ? in[0] / 255.0f : float(in[0]);
	case 5122: {
		int16_t v;
		memcpy(&v, in, 2);
		return normalized ? v / 32767.0f : float(v);
	}
	case 5123: {
		uint16_t v;
		memcpy(&v, in, 2);
		return normalized ? v / 65535.0f : float(v);
	}
	case 5125: {
		uint32_t v;
		memcpy(&v, in, 4);
		return float(v); // (the reference does not normalise 32-bit integers)
	}
	default: return 0.f;
	}
}

bool unpack_floats(const NvcGltfScene& s, long long accessor, int want_components, std::vector<float>& out)
{
	if (accessor < 0 || size_t(accessor) >= s.accessors.size())
		return false;
	const Accessor& a = s.accessors[size_t(accessor)];
	if (a.components != want_components)
		return false;
	out.resize(a.count * size_t(want_components));
	const int cs = component_size(a.component);
	for (size_t i = 0; i < a.count; ++i)
	{
		const uint8_t* e = element(s, a, i);
		if (!e)
			return false;
		for (int c = 0; c < want_components; ++c)
			out[i * want_components + c] = component_float(e + c * cs, a.component, a.normalized);
	}
	return true;
}

// ---- the reference's arithmetic ------------------------------------------------------------------------------------------

// cgltf_node_transform_local, cgltf.h:2137-2180 (column-major float[16], every product rounded to binary32)
void transform_local(const Node& n, float* lm)
{
	if (n.has_matrix)
	{
		memcpy(lm, n.matrix, sizeof(float) * 16);
		return;
	}
	const float tx = n.translation[0], ty = n.translation[1], tz = n.translation[2];
	const float qx = n.rotation[0], qy = n.rotation[1], qz = n.rotation[2], qw = n.rotation[3];
	const float sx = n.scale[0], sy = n.scale[1], sz = n.scale[2];
	lm[0] = (1 - 2 * qy * qy - 2 * qz * qz) * sx;
	lm[1] = (2 * qx * qy + 2 * qz * qw) * sx;
	lm[2] = (2 * qx * qz - 2 * qy * qw) * sx;
	lm[3] = 0.f;
	lm[4] = (2 * qx * qy - 2 * qz * qw) * sy;
	lm[5] = (1 - 2 * qx * qx - 2 * qz * qz) * sy;
	lm[6] = (2 * qy * qz + 2 * qx * qw) * sy;
	lm[7] = 0.f;
	lm[8] = (2 * qx * qz + 2 * qy * qw) * sz;
	lm[9] = (2 * qy * qz - 2 * qx * qw) * sz;
	lm[10] = (1 - 2 * qx * qx - 2 * qy * qy) * sz;
	lm[11] = 0.f;
	lm[12] = tx;
	lm[13] = ty;
	lm[14] = tz;
	lm[15] = 1.f;
}

// cgltf_node_transform_world, cgltf.h:2182-2216: local, then every ancestor's local applied on the right (3x3 + translation)
void transform_world(const std::vector<Node>& nodes, const Node& node, float* lm)
{
	transform_local(node, lm);
	long long parent = node.parent;
	int guard = 0;
	while (parent >= 0 && guard++ < 4096)
	{
		float pm[16];
		transform_local(nodes[size_t(parent)], pm);
		for (int i = 0; i < 4; ++i)
		{
			const float l0 = lm[i * 4 + 0], l1 = lm[i * 4 + 1], l2 = lm[i * 4 + 2];
			const float r0 = l0 * pm[0] + l1 * pm[4] + l2 * pm[8];
			const float r1 = l0 * pm[1] + l1 * pm[5] + l2 * pm[9];
			const float r2 = l0 * pm[2] + l1 * pm[6] + l2 * pm[10];
			lm[i * 4 + 0] = r0;
			lm[i * 4 + 1] = r1;
			lm[i * 4 + 2] = r2;
		}
		lm[12] += pm[12];
		lm[13] += pm[13];
		lm[14] += pm[14];
		parent = nodes[size_t(parent)].parent;
	}
}

// decomposeTransform, scene.cpp:295-340
void decompose(float translation[3], float rotation[4], float scale[3], const float* transform)
{
	float m[4][4];
	memcpy(m, transform, 16 * sizeof(float));
	translation[0] = m[3][0];
	translation[1] = m[3][1];
	translation[2] = m[3][2];
	const float det = m[0][0] * (m[1][1] * m[2][2] - m[2][1] * m[1][2]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
	const float sign = (det < 0.f) ? -1.f : 1.f;
	scale[0] = sqrtf(m[0][0] * m[0][0] + m[0][1] * m[0][1] + m[0][2] * m[0][2]) * sign;
	scale[1] = sqrtf(m[1][0] * m[1][0] + m[1][1] * m[1][1] + m[1][2] * m[1][2]) * sign;
	scale[2] = sqrtf(m[2][0] * m[2][0] + m[2][1] * m[2][1] + m[2][2] * m[2][2]) * sign;
	const float rsx = (scale[0] == 0.f) ? 0.f : 1.f / scale[0];
	const float rsy = (scale[1] == 0.f) ? 0.f : 1.f / scale[1];
	const float rsz = (scale[2] == 0.f) ? 0.f : 1.f / scale[2];
	const float r00 = m[0][0] * rsx, r10 = m[1][0] * rsy, r20 = m[2][0] * rsz;
	const float r01 = m[0][1] * rsx, r11 = m[1][1] * rsy, r21 = m[2][1] * rsz;
	const float r02 = m[0][2] * rsx, r12 = m[1][2] * rsy, r22 = m[2][2] * rsz;
	// Mike Day's matrix-to-quaternion conversion, branch on the largest diagonal combination
	const int qc = r22 < 0 ? (r00 > r11 ? 0 : 1) : (r00 < -r11 ? 2 : 3);
	const float qs1 = qc & 2 ? -1.f : 1.f;
	const float qs2 = qc & 1 ? -1.f : 1.f;
	const float qs3 = (qc - 1) & 2 ? -1.f : 1.f;
	const float qt = 1.f - qs3 * r00 - qs2 * r11 - qs1 * r22;
	const float qs = 0.5f / sqrtf(qt);
	rotation[qc ^ 0] = qs * qt;
	rotation[qc ^ 1] = qs * (r01 + qs1 * r10);
	rotation[qc ^ 2] = qs * (r20 + qs2 * r02);
	rotation[qc ^ 3] = qs * (r12 + qs3 * r21);
}

// meshopt_quantizeHalf (meshoptimizer.h): round-to-nearest fp16 with the library's handling of tiny / huge values
uint16_t quantize_half(float v)
{
	uint32_t ui;
	memcpy(&ui, &v, 4);
	const int s = int((ui >> 16) & 0x8000);
	const int em = int(ui & 0x7fffffff);
	int h = (em - (112 << 23) + (1 << 12)) >> 13; // bias exponent and round to nearest; 112 = 127 - 15
	h = (em < (113 << 23)) ? 0 : h;               // underflow: flush to zero; 113 encodes exponent -14
	h = (em >= (143 << 23)) ? 0x7c00 : h;         // overflow: infinity; 143 encodes exponent 16
	h = (em > (255 << 23)) ? 0x7e00 : h;          // NaN
	return uint16_t(s | h);
}

// meshopt_quantizeSnorm (meshoptimizer.h)
int quantize_snorm(float v, int bits)
{
	const float scale = float((1 << (bits - 1)) - 1);
	const float round = (v >= 0 ? 0.5f : -0.5f);
	v = (v >= -1) ? v : -1;
	v = (v <= +1) ? v : +1;
	return int(v * scale + round);
}

bool parse_float_array(const Json* j, float* out, size_t n)
{
	if (!j || j->type != Json::Array || j->size() != n)
		return false;
	for (size_t i = 0; i < n; ++i)
		out[i] = num_f(&j->at(i), 0.f);
	return true;
}

// ---- EXT_meshopt_compression / KHR_meshopt_compression ---------------------------------------------------------------------
bool is_meshopt_fallback(const Json& buffer)
{
	const Json* ext = buffer.get("extensions");
	for (const char* name : { "EXT_meshopt_compression", "KHR_meshopt_compression" })
		if (const Json* e = ext ? ext->get(name) : nullptr)
			if (const Json* f = e->get("fallback"))
				if (f->type == Json::Bool && f->b)
					return true;
	return false;
}

const Json* meshopt_extension(const Json& view)
{
	const Json* ext = view.get("extensions");
	if (!ext)
		return nullptr;
	if (const Json* e = ext->get("EXT_meshopt_compression"))
		return e;
	return ext->get("KHR_meshopt_compression");
}

enum MeshoptMode
{
	kModeInvalid,
	kModeAttributes,
	kModeTriangles,
	kModeIndices
};

struct MeshoptView
{
	size_t buffer = 0;
	uint64_t offset = 0, length = 0, stride = 0, count = 0;
	int mode = kModeInvalid;
	int filter = nvc::kFilterNone;
};

uint64_t num_u64(const Json* j)
{
	// a negative value fails every range check below, as cgltf's conversion to cgltf_size makes it huge
	return j && j->is_number() ? uint64_t((long long)(j->num)) : 0;
}

// the extension's fields (cgltf.h:5045-5130: a missing or unknown mode is invalid, an unknown filter is NONE) checked against
// cgltf_validate (cgltf.h:1640-1667), all sizes in 64 bits
int parse_meshopt_view(NvcGltfScene* s, const Json& e, const BufferView& outer, MeshoptView& m)
{
	const long long buffer = num_i(e.get("buffer"), -1);
	m.offset = num_u64(e.get("byteOffset"));
	m.length = num_u64(e.get("byteLength"));
	m.stride = num_u64(e.get("byteStride"));
	m.count = num_u64(e.get("count"));
	const Json* mode = e.get("mode");
	const std::string ms = mode && mode->type == Json::String ? mode->str : "";
	m.mode = ms == "ATTRIBUTES" ? kModeAttributes : ms == "TRIANGLES" ? kModeTriangles : ms == "INDICES" ? kModeIndices : kModeInvalid;
	const Json* filter = e.get("filter");
	const std::string fs = filter && filter->type == Json::String ? filter->str : "";
	m.filter = fs == "OCTAHEDRAL" ? nvc::kFilterOctahedral : fs == "QUATERNION" ? nvc::kFilterQuaternion : fs == "EXPONENTIAL" ? nvc::kFilterExponential : fs == "COLOR" ? nvc::kFilterColor : nvc::kFilterNone;
	if (buffer < 0 || size_t(buffer) >= s->buffers.size() || s->buffer_fallback[size_t(buffer)])
		return fail(s, NVC_ERROR_CORRUPT, "meshopt source buffer missing or without data");
	m.buffer = size_t(buffer);
	const uint64_t size = s->buffer_length[m.buffer];
	if (m.length > size || m.offset > size - m.length)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt source outside its buffer");
	if (outer.stride && outer.stride != m.stride)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt byteStride differs from the bufferView's");
	if ((m.count && m.stride > UINT64_MAX / m.count) || outer.length != m.stride * m.count)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt byteStride * count differs from the bufferView's byteLength");
	if (m.mode == kModeInvalid)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt mode");
	if (m.mode == kModeAttributes && !(m.stride % 4 == 0 && m.stride <= 256))
		return fail(s, NVC_ERROR_CORRUPT, "meshopt ATTRIBUTES stride");
	if (m.mode == kModeTriangles && m.count % 3 != 0)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt TRIANGLES count");
	if (m.mode != kModeAttributes && m.stride != 2 && m.stride != 4)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt index stride");
	if (m.mode != kModeAttributes && m.filter != nvc::kFilterNone)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt filter on an index view");
	if ((m.filter == nvc::kFilterOctahedral || m.filter == nvc::kFilterColor) && m.stride != 4 && m.stride != 8)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt filter stride");
	if (m.filter == nvc::kFilterQuaternion && m.stride != 8)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt filter stride");
	return NVC_OK;
}

// decodes one validated view into a buffer of its own and points the view at it
int decode_meshopt_view(NvcGltfScene* s, const MeshoptView& m, BufferView& view)
{
	const uint8_t* source = s->buffers[m.buffer].data() + m.offset;
	const size_t length = size_t(m.length);
	// every stream spends bytes in proportion to what it decodes (v1 vertex blocks at least their control bytes, index
	// streams a byte per triangle / index): a count the source cannot hold fails to decode, so it is refused before the
	// output is allocated
	uint64_t least = 0;
	if (m.mode == kModeAttributes)
	{
		const uint64_t per_block = m.stride ? nvc::vcodec::block_vertices(uint32_t(m.stride)) : 1;
		least = (m.count + per_block - 1) / per_block * (m.stride / 4);
	}
	else
		least = m.mode == kModeTriangles ? m.count / 3 : m.count;
	if (m.mode == kModeAttributes && m.stride == 0)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt ATTRIBUTES stride 0");
	if (m.count > 0xffffffffull || least > m.length)
		return fail(s, NVC_ERROR_CORRUPT, "meshopt count larger than its stream can hold");
	std::vector<uint8_t> out;
	try
	{
		out.resize(size_t(m.stride * m.count));
	}
	catch (const std::bad_alloc&)
	{
		return fail(s, NVC_ERROR_OUT_OF_MEMORY, "meshopt view");
	}
	const uint32_t count = uint32_t(m.count), stride = uint32_t(m.stride);
	int status = NVC_OK;
	if (m.mode == kModeAttributes)
		status = nvc::decode_vertex_stream(source, length, count, stride, out.data());
	else if (m.mode == kModeTriangles)
		status = nvc::decode_index_buffer(source, length, count, stride, out.data());
	else
		status = nvc::decode_index_sequence(source, length, count, stride, out.data());
	if (status != NVC_OK)
		return fail(s, status, "meshopt stream does not decode");
	nvc::decode_vertex_filter(m.filter, out.data(), count, stride);
	view.buffer = s->buffers.size();
	view.offset = 0;
	view.length = out.size();
	s->buffers.push_back(std::move(out));
	s->buffer_length.push_back(view.length);
	s->buffer_fallback.push_back(false);
	return NVC_OK;
}

int build(NvcGltfScene* s, const Json& root, const uint8_t* glb_bin, size_t glb_bin_size, const char* base_dir, uint32_t first_mesh_index, uint32_t material_offset)
{
	auto arr = [&](const char* key) -> const Json* {
		const Json* a = root.get(key);
		return a && a->type == Json::Array ? a : nullptr;
	};
	// ---- buffers ----
	if (const Json* a = arr("buffers"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json& b = a->at(i);
			std::vector<uint8_t> data;
			bool fallback = false;
			const Json* uri = b.get("uri");
			if (uri && uri->type == Json::String)
			{
				const std::string& u = uri->str;
				if (u.compare(0, 5, "data:") == 0)
				{
					size_t comma = u.find(',');
					if (comma == std::string::npos || u.find(";base64") == std::string::npos || !decode_base64(u.c_str() + comma + 1, u.size() - comma - 1, data))
						return fail(s, NVC_ERROR_CORRUPT, "buffer: malformed data URI");
				}
				else
				{
					std::string path = std::string(base_dir ? base_dir : "");
					if (!path.empty() && path.back() != '/')
						path += '/';
					// percent-decoding of the URI (cgltf_decode_uri)
					std::string dec;
					for (size_t k = 0; k < u.size(); ++k)
						if (u[k] == '%' && k + 2 < u.size() + 0 && isxdigit((unsigned char)u[k + 1]) && isxdigit((unsigned char)u[k + 2]))
						{
							dec.push_back(char(strtol(u.substr(k + 1, 2).c_str(), nullptr, 16)));
							k += 2;
						}
						else
							dec.push_back(u[k]);
					if (!read_file(path + dec, data))
						return fail(s, NVC_ERROR_INVALID_ARGUMENT, "buffer: cannot read " + path + dec);
				}
			}
			else if (i == 0 && glb_bin)
				data.assign(glb_bin, glb_bin + glb_bin_size);
			else if (is_meshopt_fallback(b))
				fallback = true;
			else
				return fail(s, NVC_ERROR_CORRUPT, "buffer without data");
			const long long want = num_i(b.get("byteLength"), -1);
			if (want < 0 || (!fallback && size_t(want) > data.size()))
				return fail(s, NVC_ERROR_CORRUPT, "buffer shorter than byteLength");
			s->buffers.push_back(std::move(data));
			s->buffer_length.push_back(uint64_t(want));
			s->buffer_fallback.push_back(fallback);
		}
	// ---- buffer views / accessors ----
	std::vector<std::pair<size_t, MeshoptView>> compressed; // view index, its extension
	if (const Json* a = arr("bufferViews"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json& v = a->at(i);
			BufferView bv;
			bv.buffer = size_t(num_i(v.get("buffer"), 0));
			bv.offset = size_t(num_i(v.get("byteOffset"), 0));
			bv.length = size_t(num_i(v.get("byteLength"), 0));
			bv.stride = size_t(num_i(v.get("byteStride"), 0));
			const Json* mc = meshopt_extension(v);
			// a fallback buffer has no bytes: its declared length bounds the views that a decoded stream will replace
			const uint64_t room = bv.buffer >= s->buffers.size() ? 0 : s->buffer_fallback[bv.buffer] ? s->buffer_length[bv.buffer] : s->buffers[bv.buffer].size();
			if (bv.buffer >= s->buffers.size() || bv.length > room || bv.offset > room - bv.length)
				return fail(s, NVC_ERROR_CORRUPT, "bufferView outside its buffer");
			if (s->buffer_fallback[bv.buffer] && !mc)
				return fail(s, NVC_ERROR_CORRUPT, "uncompressed bufferView in a meshopt fallback buffer");
			if (mc)
			{
				MeshoptView m;
				int status = parse_meshopt_view(s, *mc, bv, m);
				if (status != NVC_OK)
					return status;
				compressed.emplace_back(i, m);
			}
			s->views.push_back(bv);
		}
	// decompressMeshopt: every compressed view, used or not, before any accessor is read
	for (const auto& c : compressed)
	{
		int status = decode_meshopt_view(s, c.second, s->views[c.first]);
		if (status != NVC_OK)
			return status;
	}
	if (const Json* a = arr("accessors"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json& v = a->at(i);
			if (v.get("sparse"))
				return fail(s, NVC_ERROR_UNSUPPORTED, "sparse accessors are not supported");
			Accessor ac;
			ac.view = num_i(v.get("bufferView"), -1);
			ac.offset = size_t(num_i(v.get("byteOffset"), 0));
			ac.count = size_t(num_i(v.get("count"), 0));
			ac.component = int(num_i(v.get("componentType"), 0));
			const Json* n = v.get("normalized");
			ac.normalized = n && n->type == Json::Bool && n->b;
			const Json* t = v.get("type");
			const std::string ts = t && t->type == Json::String ? t->str : "";
			ac.components = ts == "SCALAR" ? 1 : ts == "VEC2" ? 2 : ts == "VEC3" ? 3 : ts == "VEC4" ? 4 : ts == "MAT2" ? 4 : ts == "MAT3" ? 9 : ts == "MAT4" ? 16 : 0;
			if (ac.components == 0 || component_size(ac.component) == 0)
				return fail(s, NVC_ERROR_CORRUPT, "accessor with unknown type");
			s->accessors.push_back(ac);
		}
	// ---- materials: only what decides postPass (scene.cpp:584-588) ----
	if (const Json* a = arr("materials"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json& m = a->at(i);
			uint8_t pp = 0;
			const Json* am = m.get("alphaMode");
			if (am && am->type == Json::String && am->str != "OPAQUE")
				pp = 1;
			if (const Json* ext = m.get("extensions"))
				if (ext->get("KHR_materials_transmission"))
					pp = 2;
			s->material_post_pass.push_back(pp);
		}
	// ---- meshes ----
	if (const Json* a = arr("meshes"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			std::vector<Primitive> prims;
			const Json* ps = a->at(i).get("primitives");
			if (ps && ps->type == Json::Array)
				for (size_t k = 0; k < ps->size(); ++k)
				{
					const Json& pj = ps->at(k);
					Primitive p;
					p.mode = int(num_i(pj.get("mode"), 4));
					p.indices = num_i(pj.get("indices"), -1);
					p.material = num_i(pj.get("material"), -1);
					if (const Json* at = pj.get("attributes"))
					{
						p.position = num_i(at->get("POSITION"), -1);
						p.normal = num_i(at->get("NORMAL"), -1);
						p.tangent = num_i(at->get("TANGENT"), -1);
						p.texcoord = num_i(at->get("TEXCOORD_0"), -1);
					}
					prims.push_back(p);
				}
			s->meshes.push_back(std::move(prims));
		}
	// ---- cameras, lights ----
	if (const Json* a = arr("cameras"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json* persp = a->at(i).get("perspective");
			s->camera_yfov.push_back(persp ? num_f(persp->get("yfov"), 0.f) : 0.f);
		}
	if (const Json* ext = root.get("extensions"))
		if (const Json* lp = ext->get("KHR_lights_punctual"))
			if (const Json* ls = lp->get("lights"))
				for (size_t i = 0; i < ls->size(); ++i)
				{
					const Json* t = ls->at(i).get("type");
					const std::string ts = t && t->type == Json::String ? t->str : "";
					s->light_type.push_back(ts == "directional" ? 1 : ts == "point" ? 2 : 0);
				}
	// ---- nodes ----
	if (const Json* a = arr("nodes"))
	{
		s->nodes.resize(a->size());
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json& nj = a->at(i);
			Node& n = s->nodes[i];
			parse_float_array(nj.get("translation"), n.translation, 3);
			parse_float_array(nj.get("rotation"), n.rotation, 4);
			parse_float_array(nj.get("scale"), n.scale, 3);
			n.has_matrix = parse_float_array(nj.get("matrix"), n.matrix, 16);
			n.mesh = num_i(nj.get("mesh"), -1);
			n.camera = num_i(nj.get("camera"), -1);
			if (const Json* ext = nj.get("extensions"))
				if (const Json* lp = ext->get("KHR_lights_punctual"))
					n.light = num_i(lp->get("light"), -1);
			if (n.mesh >= (long long)s->meshes.size() || n.camera >= (long long)s->camera_yfov.size() || n.light >= (long long)s->light_type.size())
				return fail(s, NVC_ERROR_CORRUPT, "node references a missing object");
		}
		for (size_t i = 0; i < a->size(); ++i)
			if (const Json* ch = a->at(i).get("children"))
				for (size_t k = 0; k < ch->size(); ++k)
				{
					long long c = num_i(&ch->at(k), -1);
					if (c < 0 || size_t(c) >= s->nodes.size() || s->nodes[size_t(c)].parent >= 0 || size_t(c) == i)
						return fail(s, NVC_ERROR_CORRUPT, "node hierarchy is not a forest");
					s->nodes[size_t(c)].parent = (long long)i;
				}
		// no cycles: walking up from any node must end
		for (size_t i = 0; i < s->nodes.size(); ++i)
		{
			long long p = s->nodes[i].parent;
			size_t steps = 0;
			while (p >= 0 && steps++ <= s->nodes.size())
				p = s->nodes[size_t(p)].parent;
			if (p >= 0)
				return fail(s, NVC_ERROR_CORRUPT, "node hierarchy has a cycle");
		}
	}

	// ================= loadScene, scene.cpp:497-853 =================
	// mesh scale: largest |cbrt(det(world))| over the nodes that instantiate the mesh (:503-519)
	s->mesh_scale.assign(s->meshes.size(), 1.f);
	for (const Node& n : s->nodes)
	{
		if (n.mesh < 0)
			continue;
		float xf[16];
		transform_world(s->nodes, n, xf);
		const float det = xf[0] * (xf[5] * xf[10] - xf[9] * xf[6]) - xf[1] * (xf[4] * xf[10] - xf[6] * xf[8]) + xf[2] * (xf[4] * xf[9] - xf[5] * xf[8]);
		const float scale = cbrtf(det);
		s->mesh_scale[size_t(n.mesh)] = std::max(s->mesh_scale[size_t(n.mesh)], fabsf(scale));
	}
	// primitives -> mesh indices (:521-546): only indexed triangle lists become meshes
	std::vector<std::pair<uint32_t, uint32_t>> ranges; // per glTF mesh: first mesh index (relative), count
	for (size_t i = 0; i < s->meshes.size(); ++i)
	{
		const uint32_t first = uint32_t(s->primitives.size());
		for (size_t k = 0; k < s->meshes[i].size(); ++k)
		{
			const Primitive& p = s->meshes[i][k];
			if (p.mode != 4 || p.indices < 0)
				continue;
			if (p.position < 0 || size_t(p.position) >= s->accessors.size() || size_t(p.indices) >= s->accessors.size())
				return fail(s, NVC_ERROR_CORRUPT, "primitive without POSITION / indices accessor");
			s->primitives.push_back({ uint32_t(i), uint32_t(k), &p });
		}
		ranges.emplace_back(first, uint32_t(s->primitives.size()) - first);
	}
	// draws, camera, sun (:553-633)
	std::vector<int> node_draw(s->nodes.size(), -1), node_light(s->nodes.size(), -1);
	memset(&s->info, 0, sizeof(s->info));
	s->info.camera.orientation[3] = 1.f;
	uint32_t lights = 0;
	for (size_t i = 0; i < s->nodes.size(); ++i)
	{
		const Node& n = s->nodes[i];
		if (n.mesh >= 0)
		{
			float matrix[16], translation[3], rotation[4], scale[3];
			transform_world(s->nodes, n, matrix);
			decompose(translation, rotation, scale, matrix);
			const auto range = ranges[size_t(n.mesh)];
			for (uint32_t j = 0; j < range.second; ++j)
			{
				NvcMeshDraw d;
				memset(&d, 0, sizeof(d));
				d.position[0] = translation[0], d.position[1] = translation[1], d.position[2] = translation[2];
				d.scale = cbrtf(scale[0] * scale[1] * scale[2]);
				d.orientation[0] = rotation[0], d.orientation[1] = rotation[1], d.orientation[2] = rotation[2], d.orientation[3] = rotation[3];
				d.meshIndex = first_mesh_index + range.first + j;
				const long long material = s->primitives[range.first + j].p->material;
				d.materialIndex = material >= 0 ? material_offset + uint32_t(material) : 0u;
				if (material >= 0 && size_t(material) < s->material_post_pass.size())
					d.postPass = s->material_post_pass[size_t(material)];
				node_draw[i] = int(s->draws.size());
				s->draws.push_back(d);
			}
		}
		if (n.camera >= 0)
		{
			float matrix[16], translation[3], rotation[4], scale[3];
			transform_world(s->nodes, n, matrix);
			decompose(translation, rotation, scale, matrix);
			memcpy(s->info.camera.position, translation, sizeof(translation));
			memcpy(s->info.camera.orientation, rotation, sizeof(rotation));
			s->info.camera.fovY = s->camera_yfov[size_t(n.camera)];
			s->info.has_camera = 1;
		}
		if (n.light >= 0)
		{
			float matrix[16];
			transform_world(s->nodes, n, matrix);
			if (s->light_type[size_t(n.light)] == 1)
			{
				s->info.sun_direction[0] = matrix[8], s->info.sun_direction[1] = matrix[9], s->info.sun_direction[2] = matrix[10];
				s->info.has_sun = 1;
			}
			else if (s->light_type[size_t(n.light)] == 2)
				node_light[i] = int(lights++);
		}
	}
	// animations (:713-830): one Animation per node with LINEAR T / R / S samplers of equal key count, keys baked through the hierarchy
	std::vector<const Sampler*> st(s->nodes.size(), nullptr), sr(s->nodes.size(), nullptr), ss(s->nodes.size(), nullptr);
	std::vector<std::unique_ptr<Sampler>> keep;
	if (const Json* a = arr("animations"))
		for (size_t i = 0; i < a->size(); ++i)
		{
			const Json* samplers = a->at(i).get("samplers");
			const Json* channels = a->at(i).get("channels");
			if (!samplers || !channels)
				continue;
			std::vector<Sampler*> local;
			for (size_t k = 0; k < samplers->size(); ++k)
			{
				keep.emplace_back(new Sampler());
				Sampler* sp = keep.back().get();
				sp->input = num_i(samplers->at(k).get("input"), -1);
				sp->output = num_i(samplers->at(k).get("output"), -1);
				const Json* ip = samplers->at(k).get("interpolation");
				sp->linear = !(ip && ip->type == Json::String && ip->str != "LINEAR");
				if (sp->input < 0 || sp->output < 0 || size_t(sp->input) >= s->accessors.size() || size_t(sp->output) >= s->accessors.size())
					return fail(s, NVC_ERROR_CORRUPT, "animation sampler without accessors");
				local.push_back(sp);
			}
			for (size_t k = 0; k < channels->size(); ++k)
			{
				const Json& ch = channels->at(k);
				const long long si = num_i(ch.get("sampler"), -1);
				const Json* target = ch.get("target");
				if (si < 0 || size_t(si) >= local.size() || !target)
					return fail(s, NVC_ERROR_CORRUPT, "animation channel without sampler / target");
				const long long node = num_i(target->get("node"), -1);
				if (node < 0)
					continue; // :728
				if (size_t(node) >= s->nodes.size())
					return fail(s, NVC_ERROR_CORRUPT, "animation channel targets a missing node");
				const Json* path = target->get("path");
				const std::string ps = path && path->type == Json::String ? path->str : "";
				if (ps == "translation")
					st[size_t(node)] = local[size_t(si)];
				else if (ps == "rotation")
					sr[size_t(node)] = local[size_t(si)];
				else if (ps == "scale")
					ss[size_t(node)] = local[size_t(si)];
			}
		}
	for (size_t i = 0; i < s->nodes.size(); ++i)
	{
		if (!sr[i] && !st[i] && !ss[i])
			continue;
		if (node_draw[i] == -1 && node_light[i] == -1)
			continue; // "skipping animation for node without draw or light"
		const Sampler* first = st[i] ? st[i] : sr[i] ? sr[i] : ss[i];
		const size_t keys = s->accessors[size_t(first->input)].count;
		auto count_of = [&](const Sampler* sp) { return s->accessors[size_t(sp->input)].count; };
		if ((st[i] && count_of(st[i]) != keys) || (sr[i] && count_of(sr[i]) != keys) || (ss[i] && count_of(ss[i]) != keys))
			continue; // mismatched sampler counts
		if ((st[i] && !st[i]->linear) || (sr[i] && !sr[i]->linear) || (ss[i] && !ss[i]->linear))
			continue;
		if (keys < 2)
			continue;
		std::vector<float> times, vt, vr, vs;
		if (!unpack_floats(*s, first->input, 1, times))
			return fail(s, NVC_ERROR_CORRUPT, "animation input accessor");
		if ((st[i] && (!unpack_floats(*s, st[i]->output, 3, vt) || vt.size() < keys * 3)) || (sr[i] && (!unpack_floats(*s, sr[i]->output, 4, vr) || vr.size() < keys * 4)) ||
		    (ss[i] && (!unpack_floats(*s, ss[i]->output, 3, vs) || vs.size() < keys * 3)))
			return fail(s, NVC_ERROR_CORRUPT, "animation output accessor");
		NvcAnimation an;
		an.drawIndex = node_draw[i];
		an.lightIndex = node_light[i];
		an.startTime = times[0];
		an.period = times[1] - times[0];
		an.keyframeOffset = uint32_t(s->keyframes.size());
		an.keyframeCount = uint32_t(keys);
		Node copy = s->nodes[i];
		for (size_t j = 0; j < keys; ++j)
		{
			if (st[i])
				memcpy(copy.translation, &vt[j * 3], 3 * sizeof(float));
			if (sr[i])
				memcpy(copy.rotation, &vr[j * 4], 4 * sizeof(float));
			if (ss[i])
				memcpy(copy.scale, &vs[j * 3], 3 * sizeof(float));
			float matrix[16], translation[3], rotation[4], scale[3];
			transform_world(s->nodes, copy, matrix);
			decompose(translation, rotation, scale, matrix);
			NvcKeyframe kf;
			memcpy(kf.translation, translation, sizeof(translation));
			memcpy(kf.rotation, rotation, sizeof(rotation));
			kf.scale = std::max(scale[0], std::max(scale[1], scale[2]));
			s->keyframes.push_back(kf);
		}
		s->animations.push_back(an);
	}
	s->info.node_count = uint32_t(s->nodes.size());
	s->info.mesh_count = uint32_t(s->meshes.size());
	s->info.primitive_count = uint32_t(s->primitives.size());
	s->info.draw_count = uint32_t(s->draws.size());
	s->info.animation_count = uint32_t(s->animations.size());
	s->info.keyframe_count = uint32_t(s->keyframes.size());
	s->info.material_count = uint32_t(s->material_post_pass.size());
	s->info.point_light_count = lights;
	return NVC_OK;
}

} // namespace

extern "C"
{

NVC_API int nvc_gltf_import(const void* file, size_t file_size, const char* base_dir, uint32_t first_mesh_index, uint32_t material_offset, NvcGltfScene** out_scene)
{
	if (!file || !out_scene || file_size < 4)
		return NVC_ERROR_INVALID_ARGUMENT;
	*out_scene = nullptr;
	std::unique_ptr<NvcGltfScene> s(new NvcGltfScene());
	const uint8_t* bytes = static_cast<const uint8_t*>(file);
	const char* json = reinterpret_cast<const char*>(bytes);
	size_t json_size = file_size;
	const uint8_t* bin = nullptr;
	size_t bin_size = 0;
	if (file_size >= 12 && memcmp(bytes, "glTF", 4) == 0)
	{
		// GLB container: 12-byte header, then chunks {u32 length, u32 type, data}; JSON first, BIN optional
		uint32_t version, total;
		memcpy(&version, bytes + 4, 4);
		memcpy(&total, bytes + 8, 4);
		if (version != 2 || total > file_size)
			return NVC_ERROR_CORRUPT;
		size_t at = 12;
		json = nullptr;
		while (at + 8 <= total)
		{
			uint32_t len, type;
			memcpy(&len, bytes + at, 4);
			memcpy(&type, bytes + at + 4, 4);
			at += 8;
			if (uint64_t(at) + len > total)
				return NVC_ERROR_CORRUPT;
			if (type == 0x4e4f534a && !json) // "JSON"
			{
				json = reinterpret_cast<const char*>(bytes + at);
				json_size = len;
			}
			else if (type == 0x004e4942 && !bin) // "BIN\0"
			{
				bin = bytes + at;
				bin_size = len;
			}
			at += (size_t(len) + 3) & ~size_t(3);
		}
		if (!json)
			return NVC_ERROR_CORRUPT;
	}
	JsonParser parser{ json, json + json_size };
	Json root = parser.value();
	parser.ws();
	if (!parser.ok || root.type != Json::Object)
		return NVC_ERROR_CORRUPT;
	int status = build(s.get(), root, bin, bin_size, base_dir, first_mesh_index, material_offset);
	if (status != NVC_OK)
		return status;
	*out_scene = s.release();
	return NVC_OK;
}

NVC_API void nvc_gltf_free(NvcGltfScene* scene)
{
	delete scene;
}

NVC_API int nvc_gltf_info(const NvcGltfScene* scene, NvcGltfInfo* out)
{
	if (!scene || !out)
		return NVC_ERROR_INVALID_ARGUMENT;
	*out = scene->info;
	return NVC_OK;
}

NVC_API int nvc_gltf_scene_arrays(const NvcGltfScene* scene, NvcMeshDraw* draws, NvcAnimation* animations, NvcKeyframe* keyframes, float* mesh_scale)
{
	if (!scene)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (draws && !scene->draws.empty())
		memcpy(draws, scene->draws.data(), scene->draws.size() * sizeof(NvcMeshDraw));
	if (animations && !scene->animations.empty())
		memcpy(animations, scene->animations.data(), scene->animations.size() * sizeof(NvcAnimation));
	if (keyframes && !scene->keyframes.empty())
		memcpy(keyframes, scene->keyframes.data(), scene->keyframes.size() * sizeof(NvcKeyframe));
	if (mesh_scale)
		for (size_t i = 0; i < scene->primitives.size(); ++i)
			mesh_scale[i] = scene->mesh_scale[scene->primitives[i].mesh]; // the scale appendMesh receives for this primitive
	return NVC_OK;
}

NVC_API int nvc_gltf_primitive_size(const NvcGltfScene* scene, uint32_t primitive, uint32_t* vertex_count, uint32_t* index_count)
{
	if (!scene || primitive >= scene->primitives.size() || !vertex_count || !index_count)
		return NVC_ERROR_INVALID_ARGUMENT;
	const Primitive& p = *scene->primitives[primitive].p;
	*vertex_count = uint32_t(scene->accessors[size_t(p.position)].count); // prim.attributes[0].data->count in the reference
	*index_count = uint32_t(scene->accessors[size_t(p.indices)].count);
	return NVC_OK;
}

// loadVertices (scene.cpp:342-405) + cgltf_accessor_unpack_indices: the arrays appendMesh receives
NVC_API int nvc_gltf_primitive_data(const NvcGltfScene* scene, uint32_t primitive, NvcVertex* vertices, uint32_t* indices)
{
	if (!scene || primitive >= scene->primitives.size())
		return NVC_ERROR_INVALID_ARGUMENT;
	const Primitive& p = *scene->primitives[primitive].p;
	const size_t vc = scene->accessors[size_t(p.position)].count;
	std::vector<float> scratch;
	if (vertices)
	{
		memset(vertices, 0, vc * sizeof(NvcVertex));
		if (!unpack_floats(*scene, p.position, 3, scratch))
			return NVC_ERROR_CORRUPT;
		for (size_t j = 0; j < vc; ++j)
		{
			vertices[j].vx = quantize_half(scratch[j * 3 + 0]);
			vertices[j].vy = quantize_half(scratch[j * 3 + 1]);
			vertices[j].vz = quantize_half(scratch[j * 3 + 2]);
		}
		if (p.normal >= 0)
		{
			if (!unpack_floats(*scene, p.normal, 3, scratch) || scratch.size() < vc * 3)
				return NVC_ERROR_CORRUPT;
			for (size_t j = 0; j < vc; ++j)
				vertices[j].np = uint32_t(quantize_snorm(scratch[j * 3 + 0], 10) + 511) | uint32_t(quantize_snorm(scratch[j * 3 + 1], 10) + 511) << 10 | uint32_t(quantize_snorm(scratch[j * 3 + 2], 10) + 511) << 20;
		}
		if (p.tangent >= 0)
		{
			if (!unpack_floats(*scene, p.tangent, 4, scratch) || scratch.size() < vc * 4)
				return NVC_ERROR_CORRUPT;
			for (size_t j = 0; j < vc; ++j)
			{
				const float tx = scratch[j * 4 + 0], ty = scratch[j * 4 + 1], tz = scratch[j * 4 + 2];
				const float tsum = fabsf(tx) + fabsf(ty) + fabsf(tz);
				const float tu = tz >= 0 ? tx / tsum : (1 - fabsf(ty / tsum)) * (tx >= 0 ? 1 : -1);
				const float tv = tz >= 0 ? ty / tsum : (1 - fabsf(tx / tsum)) * (ty >= 0 ? 1 : -1);
				vertices[j].tp = uint16_t((quantize_snorm(tu, 8) + 127) | (quantize_snorm(tv, 8) + 127) << 8);
				vertices[j].np |= uint32_t(scratch[j * 4 + 3] >= 0 ? 0 : 1) << 30;
			}
		}
		if (p.texcoord >= 0)
		{
			if (!unpack_floats(*scene, p.texcoord, 2, scratch) || scratch.size() < vc * 2)
				return NVC_ERROR_CORRUPT;
			for (size_t j = 0; j < vc; ++j)
			{
				vertices[j].tu = quantize_half(scratch[j * 2 + 0]);
				vertices[j].tv = quantize_half(scratch[j * 2 + 1]);
			}
		}
	}
	if (indices)
	{
		const Accessor& a = scene->accessors[size_t(p.indices)];
		if (a.components != 1 || a.component == 5126)
			return NVC_ERROR_CORRUPT;
		const int cs = component_size(a.component);
		for (size_t i = 0; i < a.count; ++i)
		{
			const uint8_t* e = element(*scene, a, i);
			if (!e)
				return NVC_ERROR_CORRUPT;
			uint32_t v = 0;
			memcpy(&v, e, size_t(cs)); // little endian: u8 / u16 / u32
			if (v >= vc)
				return NVC_ERROR_CORRUPT;
			indices[i] = v;
		}
	}
	return NVC_OK;
}

} // extern "C"
