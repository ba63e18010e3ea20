// Writes a MeshLab project (.mlp) with the reference's vendored tinyxml2, laid out as libvis' WriteMeshLabProject
// lays it out (libvis/src/libvis/external_io/meshlab_project.cc:81-111): <MeshLabProject><MeshGroup>, one <MLMesh
// label=... filename=...> per mesh holding an <MLMatrix44> whose text is a newline, then four rows of the float
// matrix printed by std::ostream, each value followed by " " and each row by a newline. Used once to produce the
// golden files tests/golden/mlp/*.mlp (tests/golden/make_mlp_golden.py); no test runs it.
//
//   mlp_writer <output.mlp> < spec
// spec: per mesh three lines: the label, the file name, and 16 row-major matrix values (parsed as float).
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "tinyxml2.h"

struct Mesh {
  std::string label, filename;
  float m[16];
};

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  std::vector<Mesh> meshes;
  std::string label, filename, values;
  while (std::getline(std::cin, label) && std::getline(std::cin, filename) && std::getline(std::cin, values)) {
    Mesh mesh;
    mesh.label = label;
    mesh.filename = filename;
    std::istringstream in(values);
    for (float& v : mesh.m) in >> v;
    if (!in) return 3;
    meshes.push_back(mesh);
  }
  tinyxml2::XMLDocument doc;
  tinyxml2::XMLElement* project = doc.NewElement("MeshLabProject");
  doc.InsertEndChild(project);
  tinyxml2::XMLElement* group = doc.NewElement("MeshGroup");
  project->InsertEndChild(group);
  for (const Mesh& mesh : meshes) {
    tinyxml2::XMLElement* element = doc.NewElement("MLMesh");
    element->SetAttribute("label", mesh.label.c_str());
    element->SetAttribute("filename", mesh.filename.c_str());
    group->InsertEndChild(element);
    tinyxml2::XMLElement* matrix = doc.NewElement("MLMatrix44");
    std::ostringstream text;
    text << std::endl;
    for (int r = 0; r < 4; ++r) {
      for (int c = 0; c < 4; ++c) text << mesh.m[4 * r + c] << " ";
      text << std::endl;
    }
    matrix->SetText(text.str().c_str());
    element->InsertEndChild(matrix);
  }
  return doc.SaveFile(argv[1]) == tinyxml2::XML_NO_ERROR ? 0 : 1;
}
