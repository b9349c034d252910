// TEST INFRASTRUCTURE (oracle/refobj/Makefile).  oracle/_ref/load_obj <in.obj> <out.bin>: the Vertex[] the reference's loadObj makes of an OBJ file
// (16-byte records, one per triangle corner, in its order), the input of appendMesh's vertex processing.  loadObj is static
// in scene.cpp, so this translation unit compiles scene.cpp itself, where it lies in the reference checkout.
#include "scene.cpp"

#include <stdio.h>

// referenced by scene.cpp's buildSceneOmm only (textures.cpp, not linked here)
unsigned char* decodeImageRGBA(const char*, int, unsigned int&, unsigned int&, unsigned int&) { return nullptr; }

int main(int argc, char** argv)
{
	if (argc != 3)
	{
		fprintf(stderr, "usage: load_obj <in.obj> <out.bin>\n");
		return 2;
	}
	std::vector<Vertex> vertices;
	if (!loadObj(vertices, argv[1]))
	{
		fprintf(stderr, "load_obj: cannot read %s\n", argv[1]);
		return 1;
	}
	FILE* f = fopen(argv[2], "wb");
	if (!f || fwrite(vertices.data(), sizeof(Vertex), vertices.size(), f) != vertices.size() || fclose(f) != 0)
	{
		fprintf(stderr, "load_obj: cannot write %s\n", argv[2]);
		return 1;
	}
	return 0;
}
