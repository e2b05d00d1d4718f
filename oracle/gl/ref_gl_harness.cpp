// TEST INFRASTRUCTURE ONLY — runs the REFERENCE's own GLSL shader files (read unmodified from <reference>/Core/Shaders at run
// time) for the mapping half of the hot path, headless, on the OpenGL 3.3 core implementation that exists in this image: Mesa 18.1.9
// llvmpipe (the software libGL that ships with Nsight Compute, an Xlib-GLX build made usable without an X server by
// oracle/gl/fake_x11.c). This is what pins oracle/efo_map.cpp: the same inputs go through these passes and through the CPU
// restatement, and tests/golden/ref_mapping_*.npz (written by tests/golden/make_gl_golden.py) holds the reference's outputs.
//
// Each function restates the HOST side of one reference pass in raw GL — the textures, formats, filters, attachments, uniforms,
// vertex attributes, transform-feedback varyings and draw calls of
//   Core/Shaders/ComputePack.cpp:37-66 (filterDepth / metriciseDepth, ElasticFusion.cpp:655-673),
//   Core/Shaders/FeedbackBuffer.cpp:30-138 + Core/GlobalModel.cpp:229-284 (first-frame map),
//   Core/IndexMap.cpp:190-258 (predictIndices), :293-476 (combinedPredict, synthesizeDepth),
//   Core/GlobalModel.cpp:356-525 (fuse: data + update), :527-671 (clean), Core/Shaders/FillIn.cpp:62-191 —
// and nothing of the shader side. Differences from the reference's host code, all forced by a core-profile context:
//   * GL_LUMINANCE* internal formats do not exist in core: R16UI / R32UI / R32F are used (the shaders read .x / .r only);
//   * transform-feedback varyings are named before linking (glTransformFeedbackVaryings) instead of
//     glTransformFeedbackVaryingsNV after it; glDrawTransformFeedback(count of the previous pass) is glDrawArrays(count);
//   * a vertex array object is bound (required in core); GL_POINT_SPRITE is always on in core and is not enabled explicitly;
//   * the 3072^2 "update map" render target is allocated at tex_dim^2 (a uniform of data.vert / update.vert), large enough for the
//     surfel counts of the fixtures;
//   * depth test on, GL_LESS: the state the reference's GUI sets for the whole application (Tools/GUI.h:68-70; SURVEY App. A-17);
//   * GLSL: resize.frag / fill_rgb.frag call texture2D() under "#version 330 core", which NVIDIA's compiler tolerates and a strict
//     core compiler rejects; for those two files the call is spelled texture() when the source is handed to the compiler
//     (efg_log() lists every such edit). Every other shader is compiled byte for byte.
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "ref_gl.h"

#define X(ret, name, args) static ret(*name) args;
EFGL_FUNCS(X)
#undef X

namespace {

std::string g_log;
void logf(const char* fmt, ...) {
  char buf[4096];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_log += buf;
  g_log += "\n";
}

struct Ctx {
  bool ok = false;
  int W = 0, H = 0, texDim = 1024;
  float fx, fy, cx, cy;
  std::string shaderDir;
  GLuint vao = 0;
  // programs
  GLuint pBilateral, pMetric, pFeedback, pInit, pIndex, pData, pUpdate, pUnstable, pCombo, pDepthSplat, pFillV, pFillN, pFillI;
  GLuint uvo = 0;
} G;

std::string read_with_includes(const std::string& dir, const std::string& file, int depth = 0) {
  std::ifstream f((dir + "/" + file).c_str());
  if (!f) {
    logf("cannot read %s/%s", dir.c_str(), file.c_str());
    return "";
  }
  std::stringstream out;
  std::string line;
  while (std::getline(f, line)) {
    if (line.compare(0, 8, "#include") == 0 && depth < 8) {  // Pangolin's GlSlProgram::PreprocessGLSL: textual insertion
      const size_t a = line.find_first_of("\"<"), b = line.find_first_of("\">", a + 1);
      out << read_with_includes(dir, line.substr(a + 1, b - a - 1), depth + 1) << "\n";
    } else {
      out << line << "\n";
    }
  }
  return out.str();
}

GLuint compile(GLenum type, const std::string& file) {
  std::string src = read_with_includes(G.shaderDir, file);
  if (src.empty()) return 0;
  if (file == "resize.frag" || file == "fill_rgb.frag") {
    size_t pos = 0, n = 0;
    while ((pos = src.find("texture2D(", pos)) != std::string::npos) {
      src.replace(pos, 10, "texture(");
      ++n;
    }
    logf("%s: %zu x texture2D( -> texture(   (GLSL 3.30 core has no texture2D)", file.c_str(), n);
  }
  GLuint s = glCreateShader(type);
  const char* p = src.c_str();
  glShaderSource(s, 1, &p, nullptr);
  glCompileShader(s);
  GLint ok = 0;
  glGetShaderiv(s, GL_COMPILE_STATUS, &ok);
  char info[4096] = {0};
  glGetShaderInfoLog(s, sizeof(info) - 1, nullptr, info);
  if (!ok) {
    logf("COMPILE FAILED %s:\n%s", file.c_str(), info);
    return 0;
  }
  if (info[0]) logf("compile log %s: %s", file.c_str(), info);
  return s;
}

GLuint program(const char* vert, const char* frag, const char* geom, bool feedback) {
  GLuint p = glCreateProgram();
  GLuint s;
  if (!(s = compile(GL_VERTEX_SHADER, vert))) return 0;
  glAttachShader(p, s);
  if (geom) {
    if (!(s = compile(GL_GEOMETRY_SHADER, geom))) return 0;
    glAttachShader(p, s);
  }
  if (frag) {
    if (!(s = compile(GL_FRAGMENT_SHADER, frag))) return 0;
    glAttachShader(p, s);
  }
  if (feedback) {  // the reference: glTransformFeedbackVaryingsNV(vPosition0, vColor0, vNormRad0, GL_INTERLEAVED_ATTRIBS)
    const char* names[3] = {"vPosition0", "vColor0", "vNormRad0"};
    glTransformFeedbackVaryings(p, 3, names, GL_INTERLEAVED_ATTRIBS);
  }
  glLinkProgram(p);
  GLint ok = 0;
  glGetProgramiv(p, GL_LINK_STATUS, &ok);
  if (!ok) {
    char info[4096] = {0};
    glGetProgramInfoLog(p, sizeof(info) - 1, nullptr, info);
    logf("LINK FAILED %s + %s + %s:\n%s", vert, frag ? frag : "-", geom ? geom : "-", info);
    return 0;
  }
  return p;
}

void u1i(GLuint p, const char* n, int v) { glUniform1i(glGetUniformLocation(p, n), v); }
void u1f(GLuint p, const char* n, float v) { glUniform1f(glGetUniformLocation(p, n), v); }
void u4f(GLuint p, const char* n, float a, float b, float c, float d) { glUniform4f(glGetUniformLocation(p, n), a, b, c, d); }
// row-major double[16] -> column-major float (Eigen::Matrix4f::data() order)
void umat(GLuint p, const char* n, const double* rowmajor) {
  float m[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) m[c * 4 + r] = (float)rowmajor[r * 4 + c];
  glUniformMatrix4fv(glGetUniformLocation(p, n), 1, GL_FALSE, m);
}
void rigid_inverse(const double* T, double* inv) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) inv[r * 4 + c] = T[c * 4 + r];
    inv[r * 4 + 3] = -(T[0 * 4 + r] * T[3] + T[1 * 4 + r] * T[7] + T[2 * 4 + r] * T[11]);
  }
  inv[12] = inv[13] = inv[14] = 0;
  inv[15] = 1;
}

// GPUTexture (Core/GPUTexture.cpp:22-40 via pangolin::GlTexture): nearest unless `linear`, clamp to edge
GLuint tex(int w, int h, GLenum internal, GLenum format, GLenum type, const void* data, bool linear = false) {
  GLuint t;
  glGenTextures(1, &t);
  glBindTexture(GL_TEXTURE_2D, t);
  glTexImage2D(GL_TEXTURE_2D, 0, (GLint)internal, w, h, 0, format, type, data);
  glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_MIN_FILTER, linear ? GL_LINEAR : GL_NEAREST);
  glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_MAG_FILTER, linear ? GL_LINEAR : GL_NEAREST);
  glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_WRAP_S, GL_CLAMP_TO_EDGE);
  glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_WRAP_T, GL_CLAMP_TO_EDGE);
  return t;
}
GLuint tex_rgb8(const uint8_t* rgb, bool linear) { return tex(G.W, G.H, GL_RGBA, GL_RGB, GL_UNSIGNED_BYTE, rgb, linear); }
GLuint tex_rgba8(const uint8_t* rgba) { return tex(G.W, G.H, GL_RGBA, GL_RGBA, GL_UNSIGNED_BYTE, rgba); }
GLuint tex_u16(const uint16_t* d) { return tex(G.W, G.H, GL_R16UI, GL_RED_INTEGER, GL_UNSIGNED_SHORT, d); }
GLuint tex_u32(const uint32_t* d) { return tex(G.W, G.H, GL_R32UI, GL_RED_INTEGER, GL_UNSIGNED_INT, d); }
GLuint tex_f32(const float* d) { return tex(G.W, G.H, GL_R32F, GL_RED, GL_FLOAT, d); }
GLuint tex_f4(const float* d, int w = 0, int h = 0) { return tex(w ? w : G.W, h ? h : G.H, GL_RGBA32F, GL_RGBA, GL_FLOAT, d); }

struct Fbo {
  GLuint fbo = 0, rb = 0;
  std::vector<GLuint> color;
  int w, h;
};
// pangolin::GlFramebuffer: AttachColour in order + AttachDepth(renderbuffer DEPTH_COMPONENT24); glDrawBuffers(all) on Bind
Fbo make_fbo(int w, int h, const std::vector<GLuint>& colors) {
  Fbo f;
  f.w = w;
  f.h = h;
  f.color = colors;
  glGenFramebuffers(1, &f.fbo);
  glBindFramebuffer(GL_FRAMEBUFFER, f.fbo);
  std::vector<GLenum> bufs;
  for (size_t i = 0; i < colors.size(); ++i) {
    glFramebufferTexture2D(GL_FRAMEBUFFER, GL_COLOR_ATTACHMENT0 + (GLenum)i, GL_TEXTURE_2D, colors[i], 0);
    bufs.push_back(GL_COLOR_ATTACHMENT0 + (GLenum)i);
  }
  glGenRenderbuffers(1, &f.rb);
  glBindRenderbuffer(GL_RENDERBUFFER, f.rb);
  glRenderbufferStorage(GL_RENDERBUFFER, GL_DEPTH_COMPONENT24, w, h);
  glFramebufferRenderbuffer(GL_FRAMEBUFFER, GL_DEPTH_ATTACHMENT, GL_RENDERBUFFER, f.rb);
  glDrawBuffers((GLsizei)bufs.size(), bufs.data());
  const GLenum st = glCheckFramebufferStatus(GL_FRAMEBUFFER);
  if (st != GL_FRAMEBUFFER_COMPLETE) logf("framebuffer incomplete: 0x%x", st);
  return f;
}
void bind_clear(const Fbo& f) {
  glBindFramebuffer(GL_FRAMEBUFFER, f.fbo);
  glViewport(0, 0, f.w, f.h);
  glClearColor(0, 0, 0, 0);
  glClear(GL_COLOR_BUFFER_BIT | GL_DEPTH_BUFFER_BIT);
}
void read_tex(GLuint t, GLenum format, GLenum type, void* out) {
  glBindTexture(GL_TEXTURE_2D, t);
  glGetTexImage(GL_TEXTURE_2D, 0, format, type, out);
}
void free_fbo(Fbo& f) {
  glBindFramebuffer(GL_FRAMEBUFFER, 0);
  glDeleteTextures((GLsizei)f.color.size(), f.color.data());
}
void del(std::initializer_list<GLuint> ts) {
  for (GLuint t : ts) glDeleteTextures(1, &t);
}

GLuint vbo_of(const void* data, size_t bytes, GLenum usage = GL_STREAM_DRAW) {
  GLuint b;
  glGenBuffers(1, &b);
  glBindBuffer(GL_ARRAY_BUFFER, b);
  glBufferData(GL_ARRAY_BUFFER, (GLsizeiptr)bytes, data, usage);
  glBindBuffer(GL_ARRAY_BUFFER, 0);
  return b;
}
// the three vec4 attributes of a surfel buffer (Vertex::SIZE = 48 bytes)
void bind_surfel_attribs(GLuint vbo) {
  glBindBuffer(GL_ARRAY_BUFFER, vbo);
  for (GLuint a = 0; a < 3; ++a) {
    glEnableVertexAttribArray(a);
    glVertexAttribPointer(a, 4, GL_FLOAT, GL_FALSE, 48, (const void*)(uintptr_t)(16 * a));
  }
}
void unbind_attribs(int n) {
  for (GLuint a = 0; a < (GLuint)n; ++a) glDisableVertexAttribArray(a);
  glBindBuffer(GL_ARRAY_BUFFER, 0);
}
// transform feedback of `draw` into a fresh buffer of cap surfels; returns primitives written and the buffer
struct Feedback {
  GLuint vbo, tfo, query;
};
Feedback begin_feedback(size_t cap_surfels) {
  Feedback f;
  std::vector<float> zeros(cap_surfels * 12, 0.f);
  f.vbo = vbo_of(zeros.data(), zeros.size() * 4);
  glGenTransformFeedbacks(1, &f.tfo);
  glGenQueries(1, &f.query);
  glBindTransformFeedback(GL_TRANSFORM_FEEDBACK, f.tfo);
  glBindBufferBase(GL_TRANSFORM_FEEDBACK_BUFFER, 0, f.vbo);
  glBeginTransformFeedback(GL_POINTS);
  glBeginQuery(GL_TRANSFORM_FEEDBACK_PRIMITIVES_WRITTEN, f.query);
  return f;
}
GLuint end_feedback(Feedback& f, float* out, size_t cap_surfels) {
  glEndTransformFeedback();
  glEndQuery(GL_TRANSFORM_FEEDBACK_PRIMITIVES_WRITTEN);
  GLuint n = 0;
  glGetQueryObjectuiv(f.query, GL_QUERY_RESULT, &n);
  glBindTransformFeedback(GL_TRANSFORM_FEEDBACK, 0);
  glFinish();
  if (n > cap_surfels) n = (GLuint)cap_surfels;
  if (out && n) {
    glBindBuffer(GL_ARRAY_BUFFER, f.vbo);
    glGetBufferSubData(GL_ARRAY_BUFFER, 0, (GLsizeiptr)n * 48, out);
    glBindBuffer(GL_ARRAY_BUFFER, 0);
  }
  return n;
}

// Mesa 18.1.9 / llvmpipe does not re-validate its rasteriser state after glDisable(GL_RASTERIZER_DISCARD): the first draw that
// follows a discard pass rasterises nothing (the second one does). One throw-away full-screen draw into a 1x1 target after every
// discard pass absorbs that; it has no bearing on what the reference's shaders compute.
void absorb_discard_quirk() {
  static GLuint src = 0, dst = 0;
  static Fbo f;
  if (!src) {
    const uint16_t one = 1000;
    src = tex(1, 1, GL_R16UI, GL_RED_INTEGER, GL_UNSIGNED_SHORT, &one);
    dst = tex(1, 1, GL_R32F, GL_RED, GL_FLOAT, nullptr);
    f = make_fbo(1, 1, {dst});
  }
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, src);
  bind_clear(f);
  glUseProgram(G.pMetric);
  u1f(G.pMetric, "maxD", 3.0f);
  glDrawArrays(GL_POINTS, 0, 1);
  glFinish();
  glBindFramebuffer(GL_FRAMEBUFFER, 0);
}

}  // namespace

extern "C" {

const char* efg_log() { return g_log.c_str(); }

// libgl: path of the Mesa libGL.so.1 (its directory and oracle/_ref/gl must be on LD_LIBRARY_PATH so libX11.so.6 resolves to the
// stand-in); shader_dir: <reference>/Core/Shaders
int efg_init(const char* libgl, const char* shader_dir, int width, int height, float fx, float fy, float cx, float cy, int tex_dim) {
  if (G.ok) return 0;
  void* x11 = dlopen("libX11.so.6", RTLD_NOW | RTLD_GLOBAL);
  if (!x11) {
    logf("libX11.so.6: %s", dlerror());
    return 1;
  }
  void* (*fake_display)(void) = (void* (*)(void))dlsym(x11, "fake_x11_display");
  unsigned long (*fake_window)(int, int) = (unsigned long (*)(int, int))dlsym(x11, "fake_x11_window");
  if (!fake_display) {
    logf("libX11.so.6 is not the stand-in (oracle/gl/fake_x11.c)");
    return 1;
  }
  void* gl = dlopen(libgl, RTLD_NOW | RTLD_GLOBAL);
  if (!gl) {
    logf("dlopen(%s): %s", libgl, dlerror());
    return 1;
  }
  typedef void* (*getproc_t)(const char*);
  getproc_t getproc = (getproc_t)dlsym(gl, "glXGetProcAddressARB");
  void* dpy = fake_display();
  void** (*chooseFB)(void*, int, const int*, int*) = (void** (*)(void*, int, const int*, int*))dlsym(gl, "glXChooseFBConfig");
  const int fb_attr[] = {0x8010, 0x1, 0x8011, 0x1, 8, 8, 9, 8, 10, 8, 12, 24, 0};
  int n = 0;
  void** cfgs = chooseFB(dpy, 0, fb_attr, &n);
  if (!cfgs || n < 1) {
    logf("no GLX framebuffer config");
    return 1;
  }
  void* (*createAttribs)(void*, void*, void*, int, const int*) = (void* (*)(void*, void*, void*, int, const int*))getproc("glXCreateContextAttribsARB");
  const int ca[] = {0x2091, 3, 0x2092, 3, 0x9126, 0x1, 0};
  void* ctx = createAttribs ? createAttribs(dpy, cfgs[0], nullptr, 1, ca) : nullptr;
  if (!ctx) {
    logf("no OpenGL 3.3 core context");
    return 1;
  }
  int (*makeCurrent)(void*, unsigned long, void*) = (int (*)(void*, unsigned long, void*))dlsym(gl, "glXMakeCurrent");
  if (!makeCurrent(dpy, fake_window(64, 64), ctx)) {
    logf("glXMakeCurrent failed");
    return 1;
  }
#define X(ret, name, args)                  \
  name = (ret(*) args)getproc(#name);       \
  if (!name) {                              \
    logf("missing GL entry point %s", #name); \
    return 1;                               \
  }
  EFGL_FUNCS(X)
#undef X
  logf("GL_RENDERER=%s GL_VERSION=%s", glGetString(0x1F01), glGetString(0x1F02));
  float pr[2] = {0, 0};
  glGetFloatv(GL_POINT_SIZE_RANGE, pr);
  logf("GL_POINT_SIZE_RANGE = %g .. %g", pr[0], pr[1]);
  G.W = width;
  G.H = height;
  G.fx = fx;
  G.fy = fy;
  G.cx = cx;
  G.cy = cy;
  G.texDim = tex_dim;
  G.shaderDir = shader_dir;
  glGenVertexArrays(1, &G.vao);
  glBindVertexArray(G.vao);
  glPixelStorei(GL_UNPACK_ALIGNMENT, 1);  // Tools/GUI.h:49-50
  glPixelStorei(GL_PACK_ALIGNMENT, 1);
  glEnable(GL_DEPTH_TEST);  // Tools/GUI.h:68-70
  glDepthFunc(GL_LESS);
  bool ok = true;
  ok &= (G.pBilateral = program("empty.vert", "depth_bilateral.frag", "quad.geom", false)) != 0;
  ok &= (G.pMetric = program("empty.vert", "depth_metric.frag", "quad.geom", false)) != 0;
  ok &= (G.pFeedback = program("vertex_feedback.vert", nullptr, "vertex_feedback.geom", true)) != 0;
  ok &= (G.pInit = program("init_unstable.vert", nullptr, nullptr, true)) != 0;
  ok &= (G.pIndex = program("index_map.vert", "index_map.frag", nullptr, false)) != 0;
  ok &= (G.pData = program("data.vert", "data.frag", "data.geom", true)) != 0;
  ok &= (G.pUpdate = program("update.vert", nullptr, nullptr, true)) != 0;
  ok &= (G.pUnstable = program("copy_unstable.vert", nullptr, "copy_unstable.geom", true)) != 0;
  ok &= (G.pCombo = program("splat.vert", "combo_splat.frag", nullptr, false)) != 0;
  ok &= (G.pDepthSplat = program("splat.vert", "depth_splat.frag", nullptr, false)) != 0;
  ok &= (G.pFillV = program("empty.vert", "fill_vertex.frag", "quad.geom", false)) != 0;
  ok &= (G.pFillN = program("empty.vert", "fill_normal.frag", "quad.geom", false)) != 0;
  ok &= (G.pFillI = program("empty.vert", "fill_rgb.frag", "quad.geom", false)) != 0;
  if (!ok) return 2;
  // uv buffer: x-major, texel centres, float (GlobalModel.cpp:101-121)
  std::vector<float> uv;
  for (int i = 0; i < width; i++)
    for (int j = 0; j < height; j++) {
      uv.push_back((float)(((float)i / (float)width) + 1.0 / (2 * (float)width)));
      uv.push_back((float)(((float)j / (float)height) + 1.0 / (2 * (float)height)));
    }
  G.uvo = vbo_of(uv.data(), uv.size() * 4, GL_STATIC_DRAW);
  G.ok = true;
  return 0;
}

// ---- ComputePack: FILTER, METRIC (ElasticFusion.cpp:655-673) ----
void efg_bilateral(const uint16_t* depth, float maxD, uint16_t* out) {
  GLuint in = tex_u16(depth), dst = tex_u16(nullptr);
  Fbo f = make_fbo(G.W, G.H, {dst});
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, in);  // input->Bind()
  bind_clear(f);
  glUseProgram(G.pBilateral);
  u1f(G.pBilateral, "cols", (float)G.W);
  u1f(G.pBilateral, "rows", (float)G.H);
  u1f(G.pBilateral, "maxD", maxD);
  glDrawArrays(GL_POINTS, 0, 1);
  glFinish();
  read_tex(dst, GL_RED_INTEGER, GL_UNSIGNED_SHORT, out);
  free_fbo(f);
  del({in});
}
void efg_metric(const uint16_t* depth, float maxD, float* out) {
  GLuint in = tex_u16(depth), dst = tex_f32(nullptr);
  Fbo f = make_fbo(G.W, G.H, {dst});
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, in);
  bind_clear(f);
  glUseProgram(G.pMetric);
  u1f(G.pMetric, "maxD", maxD);
  glDrawArrays(GL_POINTS, 0, 1);
  glFinish();
  read_tex(dst, GL_RED, GL_FLOAT, out);
  free_fbo(f);
  del({in});
}

// ---- FeedbackBuffer::compute (FeedbackBuffer.cpp:81-138): returns the number of vertices written ----
int efg_feedback(const uint8_t* rgb, const float* depth_metric, int time, float maxDepth, float* out12) {
  GLuint tc = tex_rgb8(rgb, true), td = tex_f32(depth_metric);
  glUseProgram(G.pFeedback);
  u4f(G.pFeedback, "cam", G.cx, G.cy, 1.0f / G.fx, 1.0f / G.fy);
  u1f(G.pFeedback, "threshold", 0.0f);
  u1f(G.pFeedback, "cols", (float)G.W);
  u1f(G.pFeedback, "rows", (float)G.H);
  u1i(G.pFeedback, "time", time);
  u1i(G.pFeedback, "gSampler", 0);
  u1i(G.pFeedback, "cSampler", 1);
  u1f(G.pFeedback, "maxDepth", maxDepth);
  glEnableVertexAttribArray(0);
  glBindBuffer(GL_ARRAY_BUFFER, G.uvo);
  glVertexAttribPointer(0, 2, GL_FLOAT, GL_FALSE, 0, nullptr);
  glEnable(GL_RASTERIZER_DISCARD);
  Feedback fb = begin_feedback((size_t)G.W * G.H);
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, td);
  glActiveTexture(GL_TEXTURE0 + 1);
  glBindTexture(GL_TEXTURE_2D, tc);
  glDrawArrays(GL_POINTS, 0, G.W * G.H);
  glActiveTexture(GL_TEXTURE0);
  const GLuint n = end_feedback(fb, out12, (size_t)G.W * G.H);
  glDisable(GL_RASTERIZER_DISCARD);
  unbind_attribs(1);
  del({tc, td});
  glDeleteBuffers(1, &fb.vbo);
  absorb_discard_quirk();
  return (int)n;
}

// ---- GlobalModel::initialise (GlobalModel.cpp:229-284): attribs 0,1 from the raw buffer, 2 from the filtered one; the draw
// count is the raw feedback's ("both have the same amount of vertices", which App. A-29 shows is not always so) ----
int efg_initialise(const float* raw_fb, int raw_n, const float* filt_fb, int filt_n, float* map_out) {
  const size_t cap = (size_t)G.W * G.H;
  std::vector<float> a(cap * 12, 0.f), b(cap * 12, 0.f);  // the feedback VBOs are zero-initialised and W*H vertices large
  memcpy(a.data(), raw_fb, (size_t)raw_n * 48);
  memcpy(b.data(), filt_fb, (size_t)filt_n * 48);
  GLuint va = vbo_of(a.data(), a.size() * 4), vb = vbo_of(b.data(), b.size() * 4);
  glUseProgram(G.pInit);
  glBindBuffer(GL_ARRAY_BUFFER, va);
  glEnableVertexAttribArray(0);
  glVertexAttribPointer(0, 4, GL_FLOAT, GL_FALSE, 48, nullptr);
  glEnableVertexAttribArray(1);
  glVertexAttribPointer(1, 4, GL_FLOAT, GL_FALSE, 48, (const void*)16);
  glBindBuffer(GL_ARRAY_BUFFER, vb);
  glEnableVertexAttribArray(2);
  glVertexAttribPointer(2, 4, GL_FLOAT, GL_FALSE, 48, (const void*)32);
  glEnable(GL_RASTERIZER_DISCARD);
  Feedback fb = begin_feedback(cap);
  glDrawArrays(GL_POINTS, 0, raw_n);
  const GLuint n = end_feedback(fb, map_out, cap);
  glDisable(GL_RASTERIZER_DISCARD);
  unbind_attribs(3);
  glDeleteBuffers(1, &va);
  glDeleteBuffers(1, &vb);
  glDeleteBuffers(1, &fb.vbo);
  absorb_discard_quirk();
  return (int)n;
}

// ---- IndexMap::predictIndices (IndexMap.cpp:190-258) ----
void efg_predict_indices(const float* map, int count, const double* T_wc, int time, float maxDepth, int timeDelta, uint32_t* index,
                         float* vert_conf4, float* color_time4, float* norm_rad4) {
  GLuint ti = tex_u32(nullptr), t1 = tex_f4(nullptr), t2 = tex_f4(nullptr), t3 = tex_f4(nullptr);
  Fbo f = make_fbo(G.W, G.H, {ti, t1, t2, t3});
  bind_clear(f);
  glUseProgram(G.pIndex);
  double inv[16];
  rigid_inverse(T_wc, inv);
  umat(G.pIndex, "t_inv", inv);
  u4f(G.pIndex, "cam", G.cx, G.cy, G.fx, G.fy);
  u1f(G.pIndex, "maxDepth", maxDepth);
  u1f(G.pIndex, "cols", (float)G.W);
  u1f(G.pIndex, "rows", (float)G.H);
  u1i(G.pIndex, "time", time);
  u1i(G.pIndex, "timeDelta", timeDelta);
  GLuint vbo = vbo_of(map, (size_t)(count > 0 ? count : 1) * 48);
  bind_surfel_attribs(vbo);
  glDrawArrays(GL_POINTS, 0, count);
  unbind_attribs(3);
  glFinish();
  read_tex(ti, GL_RED_INTEGER, GL_UNSIGNED_INT, index);
  read_tex(t1, GL_RGBA, GL_FLOAT, vert_conf4);
  read_tex(t2, GL_RGBA, GL_FLOAT, color_time4);
  read_tex(t3, GL_RGBA, GL_FLOAT, norm_rad4);
  free_fbo(f);
  glDeleteBuffers(1, &vbo);
}

// ---- GlobalModel::fuse (GlobalModel.cpp:356-525): the data pass (association into the update maps + transform feedback of every
// emitted vertex into newUnstableVbo) and the update pass. map is updated in place; new_out receives what the data pass fed
// back (matched measurements carry colour.w = -1, new unstable surfels -2); returns that count. ----
int efg_fuse(float* map, int count, const double* T_wc, int time, const uint8_t* rgb, const float* depth_raw, const float* depth_filt,
             const uint32_t* index, const float* vert_conf4, const float* color_time4, const float* norm_rad4, float maxDepth, float weighting,
             float* new_out) {
  const int D = G.texDim;
  GLuint u0 = tex_f4(nullptr, D, D), u1 = tex_f4(nullptr, D, D), u2 = tex_f4(nullptr, D, D);
  Fbo f = make_fbo(D, D, {u0, u1, u2});
  bind_clear(f);
  glUseProgram(G.pData);
  const char* samplers[7] = {"cSampler", "drSampler", "drfSampler", "indexSampler", "vertConfSampler", "colorTimeSampler", "normRadSampler"};
  for (int i = 0; i < 7; ++i) u1i(G.pData, samplers[i], i);
  u1f(G.pData, "time", (float)time);
  u1f(G.pData, "weighting", weighting);
  u4f(G.pData, "cam", G.cx, G.cy, (float)(1.0 / G.fx), (float)(1.0 / G.fy));
  u1f(G.pData, "cols", (float)G.W);
  u1f(G.pData, "rows", (float)G.H);
  u1f(G.pData, "scale", 1.0f);
  u1f(G.pData, "texDim", (float)D);
  umat(G.pData, "pose", T_wc);
  u1f(G.pData, "maxDepth", maxDepth);
  glEnableVertexAttribArray(0);
  glBindBuffer(GL_ARRAY_BUFFER, G.uvo);
  glVertexAttribPointer(0, 2, GL_FLOAT, GL_FALSE, 0, nullptr);
  GLuint in[7] = {tex_rgb8(rgb, true), tex_f32(depth_raw), tex_f32(depth_filt), tex_u32(index), tex_f4(vert_conf4), tex_f4(color_time4), tex_f4(norm_rad4)};
  for (int i = 0; i < 7; ++i) {
    glActiveTexture(GL_TEXTURE0 + (GLenum)i);
    glBindTexture(GL_TEXTURE_2D, in[i]);
  }
  Feedback fb = begin_feedback((size_t)G.W * G.H);
  glDrawArrays(GL_POINTS, 0, G.W * G.H);
  const GLuint n_new = end_feedback(fb, new_out, (size_t)G.W * G.H);
  glActiveTexture(GL_TEXTURE0);
  unbind_attribs(1);
  glBindFramebuffer(GL_FRAMEBUFFER, 0);
  // update pass
  glUseProgram(G.pUpdate);
  u1i(G.pUpdate, "vertSamp", 0);
  u1i(G.pUpdate, "colorSamp", 1);
  u1i(G.pUpdate, "normSamp", 2);
  u1f(G.pUpdate, "texDim", (float)D);
  u1i(G.pUpdate, "time", time);
  GLuint vbo = vbo_of(map, (size_t)(count > 0 ? count : 1) * 48);
  bind_surfel_attribs(vbo);
  glEnable(GL_RASTERIZER_DISCARD);
  Feedback fu = begin_feedback((size_t)(count > 0 ? count : 1));
  GLuint ups[3] = {u0, u1, u2};
  for (int i = 0; i < 3; ++i) {
    glActiveTexture(GL_TEXTURE0 + (GLenum)i);
    glBindTexture(GL_TEXTURE_2D, ups[i]);
  }
  glDrawArrays(GL_POINTS, 0, count);
  glActiveTexture(GL_TEXTURE0);
  end_feedback(fu, map, (size_t)count);
  glDisable(GL_RASTERIZER_DISCARD);
  unbind_attribs(3);
  free_fbo(f);
  for (int i = 0; i < 7; ++i) glDeleteTextures(1, &in[i]);
  glDeleteBuffers(1, &vbo);
  glDeleteBuffers(1, &fb.vbo);
  glDeleteBuffers(1, &fu.vbo);
  absorb_discard_quirk();
  return (int)n_new;
}

// ---- GlobalModel::clean (GlobalModel.cpp:527-671): the map, then newUnstableVbo, through copy_unstable.vert/.geom ----
int efg_clean(const float* map, int count, const float* new_unstable, int new_count, const double* T_wc, int time, const uint32_t* index,
              const float* vert_conf4, const float* color_time4, const float* norm_rad4, float confThreshold, int timeDelta, float maxDepth,
              const float* nodes16, int n_nodes, const float* depth, int isFern, float* out) {
  glUseProgram(G.pUnstable);
  u1i(G.pUnstable, "time", time);
  u1f(G.pUnstable, "confThreshold", confThreshold);
  u1f(G.pUnstable, "scale", 1.0f);
  const char* samplers[6] = {"indexSampler", "vertConfSampler", "colorTimeSampler", "normRadSampler", "nodeSampler", "depthSampler"};
  for (int i = 0; i < 6; ++i) u1i(G.pUnstable, samplers[i], i);
  // GlobalModel::NODE_TEXTURE_DIMENSION is 16384 (GlobalModel.cpp:25); llvmpipe's GL_MAX_TEXTURE_SIZE is 8192, so the node texture
  // is 8192 texels wide here (512 nodes) -- its width reaches the shader only through the `nodeCols` uniform set from it.
  const int NODE_DIM = 8192;
  u1f(G.pUnstable, "nodes", (float)n_nodes);
  u1f(G.pUnstable, "nodeCols", (float)NODE_DIM);
  u1i(G.pUnstable, "timeDelta", timeDelta);
  u1f(G.pUnstable, "maxDepth", maxDepth);
  u1i(G.pUnstable, "isFern", isFern);
  double inv[16];
  rigid_inverse(T_wc, inv);
  umat(G.pUnstable, "t_inv", inv);
  u4f(G.pUnstable, "cam", G.cx, G.cy, G.fx, G.fy);
  u1f(G.pUnstable, "cols", (float)G.W);
  u1f(G.pUnstable, "rows", (float)G.H);
  std::vector<float> nodebuf(NODE_DIM, 0.f);
  if (n_nodes > 0) memcpy(nodebuf.data(), nodes16, (size_t)n_nodes * 64);
  std::vector<float> zdepth;
  if (!depth) {
    zdepth.assign((size_t)G.W * G.H, 0.f);
    depth = zdepth.data();
  }
  GLuint in[6] = {tex_u32(index), tex_f4(vert_conf4), tex_f4(color_time4), tex_f4(norm_rad4),
                  tex(NODE_DIM, 1, GL_R32F, GL_RED, GL_FLOAT, nodebuf.data()), tex_f32(depth)};
  for (int i = 0; i < 6; ++i) {
    glActiveTexture(GL_TEXTURE0 + (GLenum)i);
    glBindTexture(GL_TEXTURE_2D, in[i]);
  }
  glActiveTexture(GL_TEXTURE0);
  const size_t cap = (size_t)count + new_count + 1;
  GLuint va = vbo_of(map, (size_t)(count > 0 ? count : 1) * 48), vb = vbo_of(new_unstable, (size_t)(new_count > 0 ? new_count : 1) * 48);
  glEnable(GL_RASTERIZER_DISCARD);
  Feedback fb = begin_feedback(cap);
  bind_surfel_attribs(va);
  glDrawArrays(GL_POINTS, 0, count);
  bind_surfel_attribs(vb);
  glDrawArrays(GL_POINTS, 0, new_count);
  const GLuint n = end_feedback(fb, out, cap);
  glDisable(GL_RASTERIZER_DISCARD);
  unbind_attribs(3);
  for (int i = 0; i < 6; ++i) glDeleteTextures(1, &in[i]);
  glDeleteBuffers(1, &va);
  glDeleteBuffers(1, &vb);
  glDeleteBuffers(1, &fb.vbo);
  absorb_discard_quirk();
  return (int)n;
}

// ---- IndexMap::combinedPredict / synthesizeDepth (IndexMap.cpp:293-476) ----
void efg_combined_predict(const float* map, int count, const double* T_wc, float maxDepth, float confThreshold, int time, int maxTime,
                          int timeDelta, uint8_t* image4, float* vertex4, float* normal4, uint16_t* time_out, float* depth_out, int depth_only) {
  glEnable(GL_PROGRAM_POINT_SIZE);
  const GLuint p = depth_only ? G.pDepthSplat : G.pCombo;
  Fbo f;
  GLuint ti = 0, tv = 0, tn = 0, tt = 0, td = 0;
  if (depth_only) {
    td = tex_f32(nullptr);
    f = make_fbo(G.W, G.H, {td});
  } else {
    ti = tex_rgb8(nullptr, false);
    tv = tex_f4(nullptr);
    tn = tex_f4(nullptr);
    tt = tex_u16(nullptr);
    f = make_fbo(G.W, G.H, {ti, tv, tn, tt});
  }
  bind_clear(f);
  glUseProgram(p);
  double inv[16];
  rigid_inverse(T_wc, inv);
  umat(p, "t_inv", inv);
  u4f(p, "cam", G.cx, G.cy, G.fx, G.fy);
  u1f(p, "maxDepth", maxDepth);
  u1f(p, "confThreshold", confThreshold);
  u1f(p, "cols", (float)G.W);
  u1f(p, "rows", (float)G.H);
  u1i(p, "time", time);
  u1i(p, "maxTime", maxTime);
  u1i(p, "timeDelta", timeDelta);
  GLuint vbo = vbo_of(map, (size_t)(count > 0 ? count : 1) * 48);
  bind_surfel_attribs(vbo);
  glDrawArrays(GL_POINTS, 0, count);
  unbind_attribs(3);
  glFinish();
  if (depth_only) {
    read_tex(td, GL_RED, GL_FLOAT, depth_out);
  } else {
    read_tex(ti, GL_RGBA, GL_UNSIGNED_BYTE, image4);
    read_tex(tv, GL_RGBA, GL_FLOAT, vertex4);
    read_tex(tn, GL_RGBA, GL_FLOAT, normal4);
    read_tex(tt, GL_RED_INTEGER, GL_UNSIGNED_SHORT, time_out);
  }
  free_fbo(f);
  glDeleteBuffers(1, &vbo);
  glDisable(GL_PROGRAM_POINT_SIZE);
}

// ---- FillIn::vertex / normal / image (FillIn.cpp:62-191) ----
static void fill_geom(GLuint p, const float* existing4, const uint16_t* raw_depth, int passthrough, float* out4) {
  GLuint te = tex_f4(existing4), tr = tex_u16(raw_depth), dst = tex_f4(nullptr);
  Fbo f = make_fbo(G.W, G.H, {dst});
  bind_clear(f);
  glUseProgram(p);
  u1i(p, "eSampler", 0);
  u1i(p, "rSampler", 1);
  u1i(p, "passthrough", passthrough);
  u4f(p, "cam", G.cx, G.cy, 1.0f / G.fx, 1.0f / G.fy);
  u1f(p, "cols", (float)G.W);
  u1f(p, "rows", (float)G.H);
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, te);
  glActiveTexture(GL_TEXTURE0 + 1);
  glBindTexture(GL_TEXTURE_2D, tr);
  glDrawArrays(GL_POINTS, 0, 1);
  glActiveTexture(GL_TEXTURE0);
  glFinish();
  read_tex(dst, GL_RGBA, GL_FLOAT, out4);
  free_fbo(f);
  del({te, tr});
}
void efg_fill_vertex(const float* existing4, const uint16_t* raw_depth, int passthrough, float* out4) { fill_geom(G.pFillV, existing4, raw_depth, passthrough, out4); }
void efg_fill_normal(const float* existing4, const uint16_t* raw_depth, int passthrough, float* out4) { fill_geom(G.pFillN, existing4, raw_depth, passthrough, out4); }
void efg_fill_image(const uint8_t* existing4, const uint8_t* rgb, int passthrough, uint8_t* out4) {
  GLuint te = tex_rgba8(existing4), tr = tex_rgb8(rgb, true), dst = tex_rgb8(nullptr, false);
  Fbo f = make_fbo(G.W, G.H, {dst});
  bind_clear(f);
  glUseProgram(G.pFillI);
  u1i(G.pFillI, "eSampler", 0);
  u1i(G.pFillI, "rSampler", 1);
  u1i(G.pFillI, "passthrough", passthrough);
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, te);
  glActiveTexture(GL_TEXTURE0 + 1);
  glBindTexture(GL_TEXTURE_2D, tr);
  glDrawArrays(GL_POINTS, 0, 1);
  glActiveTexture(GL_TEXTURE0);
  glFinish();
  read_tex(dst, GL_RGBA, GL_UNSIGNED_BYTE, out4);
  free_fbo(f);
  del({te, tr});
}

// ---- Resize::image / vertex / time (Resize.cpp:50-159): empty.vert + quad.geom + resize.frag into a (W/factor) x (H/factor)
// target. which: 0 = RGBA8 image (read back as RGB, 3 bytes per texel), 1 = RGBA32F, 2 = R16UI through the float sampler
// (formally undefined; reported as read back) ----
static GLuint g_pResize = 0;
void efg_resize(const void* src, int which, int factor, void* out) {
  if (!g_pResize) g_pResize = program("empty.vert", "resize.frag", "quad.geom", false);
  const int dw = G.W / factor, dh = G.H / factor;
  GLuint ts = which == 0 ? tex_rgba8((const uint8_t*)src) : which == 1 ? tex_f4((const float*)src) : tex_u16((const uint16_t*)src);
  GLuint dst = which == 0 ? tex(dw, dh, GL_RGBA, GL_RGB, GL_UNSIGNED_BYTE, nullptr)
                          : which == 1 ? tex(dw, dh, GL_RGBA32F, GL_RGBA, GL_FLOAT, nullptr) : tex(dw, dh, GL_R16UI, GL_RED_INTEGER, GL_UNSIGNED_SHORT, nullptr);
  Fbo f = make_fbo(dw, dh, {dst});
  bind_clear(f);
  glUseProgram(g_pResize);
  u1i(g_pResize, "eSampler", 0);
  glActiveTexture(GL_TEXTURE0);
  glBindTexture(GL_TEXTURE_2D, ts);
  glDrawArrays(GL_POINTS, 0, 1);
  glFinish();
  if (which == 0)
    glReadPixels(0, 0, dw, dh, GL_RGB, GL_UNSIGNED_BYTE, out);
  else if (which == 1)
    glReadPixels(0, 0, dw, dh, GL_RGBA, GL_FLOAT, out);
  else
    glReadPixels(0, 0, dw, dh, GL_RED_INTEGER, GL_UNSIGNED_SHORT, out);
  free_fbo(f);
  del({ts});
}

unsigned efg_gl_error() { return glGetError(); }

}  // extern "C"
