// TEST INFRASTRUCTURE ONLY — the REFERENCE's global-surface shaders (draw_global_surface.vert / .geom with .frag or _phong.frag,
// read unmodified from <reference>/Core/Shaders at run time) drawn headless on Mesa llvmpipe, in the GL context that
// oracle/gl/ref_gl_harness.cpp (efg_init) made current. Built on first use by oracle/ef_refgl_render.py; its outputs are
// tests/golden/ref_render_*.npz (tests/golden/make_render_golden.py).
//
// Restates the HOST side of GlobalModel::renderPointCloud (Core/GlobalModel.cpp:286-350, drawPoints = false) and of the colour pass
// of GUI::drawFXAA (Tools/GUI.h:273-345): uniforms, the three vec4 surfel attributes (Vertex::SIZE = 48 bytes) and one point per
// surfel, into an RGBA8 + DEPTH_COMPONENT24 target cleared to (0,0,0,0) and depth 1, GL_LESS (the state the reference's GUI sets for
// the whole application, Tools/GUI.h:68-70), read back with glReadPixels (row 0 = window y 0). The shaders' #include is resolved by
// textual insertion, as Pangolin's GlSlProgram::PreprocessGLSL does; nothing of the shader side is edited.
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <fstream>
#include <sstream>
#include <string>

#include "ref_gl.h"

#define X(ret, name, args) static ret(*name) args;
EFGL_FUNCS(X)
#undef X
static void (*glUniform3f)(GLint, GLfloat, GLfloat, GLfloat);

namespace {

std::string g_log, g_dir;
GLuint g_prog[2] = {0, 0};

std::string read_with_includes(const std::string& file, int depth = 0) {
  std::ifstream f((g_dir + "/" + file).c_str());
  if (!f) {
    g_log += "cannot read " + g_dir + "/" + file + "\n";
    return "";
  }
  std::stringstream out;
  std::string line;
  while (std::getline(f, line)) {
    if (line.compare(0, 8, "#include") == 0 && depth < 8) {
      const size_t a = line.find_first_of("\"<"), b = line.find_first_of("\">", a + 1);
      out << read_with_includes(line.substr(a + 1, b - a - 1), depth + 1) << "\n";
    } else {
      out << line << "\n";
    }
  }
  return out.str();
}

GLuint compile(GLenum type, const char* file) {
  const std::string src = read_with_includes(file);
  if (src.empty()) return 0;
  GLuint s = glCreateShader(type);
  const char* p = src.c_str();
  glShaderSource(s, 1, &p, nullptr);
  glCompileShader(s);
  GLint ok = 0;
  glGetShaderiv(s, GL_COMPILE_STATUS, &ok);
  if (!ok) {
    char info[4096] = {0};
    glGetShaderInfoLog(s, sizeof(info) - 1, nullptr, info);
    g_log += std::string("COMPILE FAILED ") + file + ":\n" + info + "\n";
    return 0;
  }
  return s;
}

GLuint program(bool phong) {
  const GLuint v = compile(GL_VERTEX_SHADER, "draw_global_surface.vert"), g = compile(GL_GEOMETRY_SHADER, "draw_global_surface.geom"),
               f = compile(GL_FRAGMENT_SHADER, phong ? "draw_global_surface_phong.frag" : "draw_global_surface.frag");
  if (!v || !g || !f) return 0;
  GLuint p = glCreateProgram();
  glAttachShader(p, v);
  glAttachShader(p, g);
  glAttachShader(p, f);
  glLinkProgram(p);
  GLint ok = 0;
  glGetProgramiv(p, GL_LINK_STATUS, &ok);
  if (!ok) {
    char info[4096] = {0};
    glGetProgramInfoLog(p, sizeof(info) - 1, nullptr, info);
    g_log += std::string("LINK FAILED:\n") + info + "\n";
    return 0;
  }
  return p;
}

bool load(const char* libgl) {
  void* gl = dlopen(libgl, RTLD_NOW | RTLD_NOLOAD);
  if (!gl) {
    g_log += std::string("libGL is not loaded (initialise the harness first): ") + libgl + "\n";
    return false;
  }
  typedef void* (*getproc_t)(const char*);
  getproc_t getproc = (getproc_t)dlsym(gl, "glXGetProcAddressARB");
#define X(ret, name, args)                                              \
  name = (ret(*) args)getproc(#name);                                   \
  if (!name) {                                                          \
    g_log += std::string("missing GL entry point ") + #name + "\n";     \
    return false;                                                       \
  }
  EFGL_FUNCS(X)
  X(void, glUniform3f, (GLint, GLfloat, GLfloat, GLfloat))
#undef X
  return true;
}

void u1i(GLuint p, const char* n, int v) { glUniform1i(glGetUniformLocation(p, n), v); }
void u1f(GLuint p, const char* n, float v) { glUniform1f(glGetUniformLocation(p, n), v); }

}  // namespace

extern "C" {

const char* efgr_log() { return g_log.c_str(); }

// map: count surfels of 12 floats; mvp / mv: column-major float[16]; rgba_out: width * height * 4 bytes. 0 on success.
int efgr_render(const char* libgl, const char* shader_dir, const float* map, int count, int width, int height, const float* mvp, const float* mv,
                float threshold, int colorType, int unstable, int drawWindow, int time, int timeDelta, int phong, float signMult,
                uint8_t* rgba_out) {
  if (!glCreateShader && !load(libgl)) return 1;
  g_dir = shader_dir;
  GLuint& p = g_prog[phong ? 1 : 0];
  if (!p) p = program(phong != 0);
  if (!p) return 2;
  // target: RGBA8 colour texture + DEPTH_COMPONENT24 renderbuffer (pangolin::GlFramebuffer + GlRenderBuffer)
  GLuint tex, fbo, rb, vbo;
  glGenTextures(1, &tex);
  glBindTexture(GL_TEXTURE_2D, tex);
  glTexImage2D(GL_TEXTURE_2D, 0, GL_RGBA8, width, height, 0, GL_RGBA, GL_UNSIGNED_BYTE, nullptr);
  glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_MIN_FILTER, GL_NEAREST);
  glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_MAG_FILTER, GL_NEAREST);
  glGenFramebuffers(1, &fbo);
  glBindFramebuffer(GL_FRAMEBUFFER, fbo);
  glFramebufferTexture2D(GL_FRAMEBUFFER, GL_COLOR_ATTACHMENT0, GL_TEXTURE_2D, tex, 0);
  glGenRenderbuffers(1, &rb);
  glBindRenderbuffer(GL_RENDERBUFFER, rb);
  glRenderbufferStorage(GL_RENDERBUFFER, GL_DEPTH_COMPONENT24, width, height);
  glFramebufferRenderbuffer(GL_FRAMEBUFFER, GL_DEPTH_ATTACHMENT, GL_RENDERBUFFER, rb);
  const GLenum buf = GL_COLOR_ATTACHMENT0;
  glDrawBuffers(1, &buf);
  if (glCheckFramebufferStatus(GL_FRAMEBUFFER) != GL_FRAMEBUFFER_COMPLETE) {
    g_log += "framebuffer incomplete\n";
    return 3;
  }
  glViewport(0, 0, width, height);
  glEnable(GL_DEPTH_TEST);
  glDepthFunc(GL_LESS);
  glPixelStorei(GL_PACK_ALIGNMENT, 1);
  glClearColor(0, 0, 0, 0);
  glClear(GL_COLOR_BUFFER_BIT | GL_DEPTH_BUFFER_BIT);
  glUseProgram(p);
  glUniformMatrix4fv(glGetUniformLocation(p, "MVP"), 1, GL_FALSE, mvp);
  u1f(p, "threshold", threshold);
  u1i(p, "colorType", colorType);
  u1i(p, "unstable", unstable);
  u1i(p, "drawWindow", drawWindow);
  u1i(p, "time", time);
  u1i(p, "timeDelta", timeDelta);
  if (phong) {
    u1f(p, "signMult", signMult);
    glUniform3f(glGetUniformLocation(p, "lightpos"), mv[12], mv[13], mv[14]);  // modelView.topRightCorner(3, 1)
  }
  glGenBuffers(1, &vbo);
  glBindBuffer(GL_ARRAY_BUFFER, vbo);
  glBufferData(GL_ARRAY_BUFFER, (GLsizeiptr)(count > 0 ? count : 1) * 48, map, GL_STREAM_DRAW);
  for (GLuint a = 0; a < 3; ++a) {
    glEnableVertexAttribArray(a);
    glVertexAttribPointer(a, 4, GL_FLOAT, GL_FALSE, 48, (const void*)(uintptr_t)(16 * a));
  }
  glDrawArrays(GL_POINTS, 0, count);
  for (GLuint a = 0; a < 3; ++a) glDisableVertexAttribArray(a);
  glBindBuffer(GL_ARRAY_BUFFER, 0);
  glFinish();
  glReadPixels(0, 0, width, height, GL_RGBA, GL_UNSIGNED_BYTE, rgba_out);
  glBindFramebuffer(GL_FRAMEBUFFER, 0);
  glDeleteTextures(1, &tex);
  glDeleteBuffers(1, &vbo);
  return glGetError() == 0 ? 0 : 4;
}

}  // extern "C"
