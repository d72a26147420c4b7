// mhb_main.cpp -- `megahit_core` drop-in for the SdBG-construction sub-commands.
//
// Mirrors the dispatch surface of voutcn/megahit src/main.cpp:68-110: `buildlib` (plain-text inputs), `count` and `seq2sdbg` run on the
// GPU through libmhb (same option names as src/main_sdbg_build.cpp:42-57 and :164-189, same files);
// `checkcpu`/`checkpopcnt`/`checkbmi2`/`dumpversion`/`kmax` answer as the reference does so that the
// Python driver (src/megahit:612-629) accepts the binary; every other sub-command is forwarded to the
// reference binary named by $MHB_REFERENCE_CORE (or `megahit_core_ref` next to this executable).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <fcntl.h>
#include <sys/resource.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <unistd.h>

#include <algorithm>
#include <fstream>
#include <map>
#include <string>
#include <vector>

#include "mhb.h"

namespace {

struct Opt {
  const char *long_name, *short_name;
  bool is_flag;
};

// getopt_long-like parsing as utils/options_description.cpp:33-96: "--name value", "--name=value", "-s value"
bool parse(int argc, char **argv, const std::vector<Opt> &opts, std::map<std::string, std::string> *out, std::string *err) {
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i], name, value;
    bool has_value = false;
    if (a.rfind("--", 0) == 0) {
      name = a.substr(2);
      const size_t eq = name.find('=');
      if (eq != std::string::npos) {
        value = name.substr(eq + 1);
        name = name.substr(0, eq);
        has_value = true;
      }
    } else if (a.size() >= 2 && a[0] == '-') {
      const std::string s = a.substr(1, 1);
      for (const auto &o : opts)
        if (o.short_name[0] && s == o.short_name) name = o.long_name;
      if (name.empty()) {
        *err = "invalid option -- '" + s + "'";
        return false;
      }
      if (a.size() > 2) {
        value = a.substr(2);
        has_value = true;
      }
    } else {
      continue;  // positional arguments are ignored, as getopt_long permutes them away
    }
    const Opt *found = nullptr;
    for (const auto &o : opts)
      if (name == o.long_name) found = &o;
    if (!found) {
      *err = "unrecognized option '--" + name + "'";
      return false;
    }
    if (found->is_flag) {
      (*out)[name] = "1";
    } else {
      if (!has_value) {
        if (i + 1 >= argc) {
          *err = "option '--" + name + "' requires an argument";
          return false;
        }
        value = argv[++i];
      }
      (*out)[name] = value;
    }
  }
  return true;
}

struct RssRecorder {  // utils.h:128-157 AutoMaxRssRecorder
  timeval t0;
  RssRecorder() { gettimeofday(&t0, nullptr); }
  ~RssRecorder() {
    timeval t1;
    gettimeofday(&t1, nullptr);
    rusage u;
    getrusage(RUSAGE_SELF, &u);
    fprintf(stderr, "INFO  %-30s: %4d - Real: %.4f\tuser: %.4f\tsys: %.4f\tmaxrss: %ld\n", "megahit_b200", __LINE__,
            (t1.tv_sec - t0.tv_sec) + (t1.tv_usec - t0.tv_usec) * 1e-6, u.ru_utime.tv_sec + u.ru_utime.tv_usec * 1e-6,
            u.ru_stime.tv_sec + u.ru_stime.tv_usec * 1e-6, u.ru_maxrss);
  }
};

int fail_usage(const std::string &msg, const char *usage) {
  fprintf(stderr, "%s\n%s\n", msg.c_str(), usage);
  return 1;
}

int main_count(int argc, char **argv) {
  RssRecorder rec;
  const std::vector<Opt> opts = {{"kmer_k", "k", false},          {"min_kmer_frequency", "m", false}, {"host_mem", "", false},
                                 {"num_cpu_threads", "", false},  {"read_lib_file", "", false},       {"output_prefix", "", false},
                                 {"mem_flag", "", false},         {"gpus", "", false}};
  const char *usage = "Usage: sdbg_builder count --input_file fastx_file -o out";
  std::map<std::string, std::string> v;
  std::string err;
  if (!parse(argc, argv, opts, &v, &err)) return fail_usage(err, usage);
  mhb_count_opts o;
  memset(&o, 0, sizeof(o));
  o.k = v.count("kmer_k") ? (uint32_t)atoi(v["kmer_k"].c_str()) : 21;  // kmer_counter.h:37-43 defaults
  o.m = v.count("min_kmer_frequency") ? atoi(v["min_kmer_frequency"].c_str()) : 2;
  o.host_mem = v.count("host_mem") ? atof(v["host_mem"].c_str()) : 0;
  o.num_cpu_threads = v.count("num_cpu_threads") ? atoi(v["num_cpu_threads"].c_str()) : 0;
  o.mem_flag = v.count("mem_flag") ? atoi(v["mem_flag"].c_str()) : 1;
  const std::string lib = v["read_lib_file"], out = v.count("output_prefix") ? v["output_prefix"] : "out";
  o.read_lib_file = lib.c_str();
  o.output_prefix = out.c_str();
  if (lib.empty()) return fail_usage("No read library configuration file!", usage);
  if (o.host_mem == 0) return fail_usage("Please specify the host memory!", usage);
  // --gpus N / MHB_GPUS=N (not an option of the reference, which the Python driver never passes): one worker per GPU
  const int gpus = v.count("gpus") ? atoi(v["gpus"].c_str()) : (getenv("MHB_GPUS") ? atoi(getenv("MHB_GPUS")) : 1);
  if (int rc = gpus > 1 ? mhb_count_run_multi(&o, gpus) : mhb_count_run(&o)) {
    fprintf(stderr, "FATAL megahit_b200: %s\n", mhb_last_error());
    (void)rc;
    exit(1);
  }
  return 0;
}

int main_seq2sdbg(int argc, char **argv) {
  RssRecorder rec;
  const std::vector<Opt> opts = {{"host_mem", "", false},     {"kmer_size", "k", false},    {"kmer_from", "", false},
                                 {"num_cpu_threads", "t", false}, {"contig", "", false},    {"bubble", "", false},
                                 {"addi_contig", "", false},  {"local_contig", "", false},  {"input_prefix", "", false},
                                 {"output_prefix", "o", false}, {"need_mercy", "", true},   {"mem_flag", "", false},
                                 {"gpus", "", false}};
  const char *usage =
      "Usage: sdbg_builder seq2sdbg -k kmer_size --contig contigs.fa [--addi_contig add.fa] [--input_prefix input] -o out";
  std::map<std::string, std::string> v;
  std::string err;
  if (!parse(argc, argv, opts, &v, &err)) return fail_usage(err, usage);
  mhb_seq2sdbg_opts o;
  memset(&o, 0, sizeof(o));
  o.host_mem = v.count("host_mem") ? atof(v["host_mem"].c_str()) : 0;
  o.k = v.count("kmer_size") ? (uint32_t)atoi(v["kmer_size"].c_str()) : 0;
  o.k_from = v.count("kmer_from") ? (uint32_t)atoi(v["kmer_from"].c_str()) : 0;
  o.num_cpu_threads = v.count("num_cpu_threads") ? atoi(v["num_cpu_threads"].c_str()) : 0;
  o.mem_flag = v.count("mem_flag") ? atoi(v["mem_flag"].c_str()) : 1;
  o.need_mercy = v.count("need_mercy") ? 1 : 0;
  const std::string contig = v["contig"], bubble = v["bubble"], addi = v["addi_contig"], local = v["local_contig"],
                    in = v["input_prefix"], out = v["output_prefix"];
  o.contig = contig.c_str();
  o.bubble = bubble.c_str();
  o.addi_contig = addi.c_str();
  o.local_contig = local.c_str();
  o.input_prefix = in.c_str();
  o.output_prefix = out.c_str();
  if (in.empty() && contig.empty() && addi.empty()) return fail_usage("No input files!", usage);
  if (o.k < 9) return fail_usage("kmer size must be >= 9!", usage);
  if (o.host_mem == 0) return fail_usage("Please specify the host memory!", usage);
  // --gpus N / MHB_GPUS=N (not an option of the reference, which the Python driver never passes): one worker per GPU
  const int gpus = v.count("gpus") ? atoi(v["gpus"].c_str()) : (getenv("MHB_GPUS") ? atoi(getenv("MHB_GPUS")) : 1);
  if (int rc = gpus > 1 ? mhb_seq2sdbg_run_multi(&o, gpus) : mhb_seq2sdbg_run(&o)) {
    fprintf(stderr, "FATAL megahit_b200: %s\n", mhb_last_error());
    (void)rc;
    exit(1);
  }
  return 0;
}

int forward_to_reference(char **argv);

// argv without the option `name` (in the "--name value" and "--name=value" forms `parse` takes), walked as `parse` walks
// it so that an option's value is never mistaken for an option; argv[0] and argv[1] (the sub-command) are kept
std::vector<char *> drop_option(int argc, char **argv, const std::vector<Opt> &opts, const std::string &name) {
  std::vector<char *> out(argv, argv + std::min(argc, 2));
  for (int i = 2; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--" + name) {
      ++i;  // and its value
      continue;
    }
    if (a.rfind("--" + name + "=", 0) == 0) continue;
    out.push_back(argv[i]);
    bool takes_next = false;  // a value-taking option whose value is the next argument
    if (a.rfind("--", 0) == 0) {
      if (a.find('=') == std::string::npos)
        for (const auto &o : opts)
          if (a.substr(2) == o.long_name) takes_next = !o.is_flag;
    } else if (a.size() == 2 && a[0] == '-') {
      for (const auto &o : opts)
        if (o.short_name[0] && a.substr(1) == o.short_name) takes_next = !o.is_flag;
    }
    if (takes_next && i + 1 < argc) out.push_back(argv[++i]);
  }
  out.push_back(nullptr);
  return out;
}

// main_iterate (main_iterate.cpp:57-112, 196-221)
int main_iterate(int argc, char **argv, char **full_argv) {
  RssRecorder rec;
  const std::vector<Opt> opts = {{"contig_file", "c", false}, {"bubble_file", "b", false},     {"read_file", "r", false},
                                 {"num_cpu_threads", "t", false}, {"kmer_k", "k", false},       {"step", "s", false},
                                 {"output_prefix", "o", false}, {"gpus", "", false}};
  const char *usage = "Usage: megahit_core iterate [opt]\nopt with (*) are must";
  std::map<std::string, std::string> v;
  std::string err;
  if (!parse(argc, argv, opts, &v, &err)) return fail_usage(err, usage);
  mhb_iterate_opts o;
  memset(&o, 0, sizeof(o));
  const std::string c = v["contig_file"], b = v["bubble_file"], r = v["read_file"], out = v["output_prefix"];
  o.contig_file = c.c_str();
  o.bubble_file = b.c_str();
  o.read_file = r.c_str();
  o.output_prefix = out.c_str();
  o.num_cpu_threads = v.count("num_cpu_threads") ? atoi(v["num_cpu_threads"].c_str()) : 0;
  const int k = v.count("kmer_k") ? atoi(v["kmer_k"].c_str()) : 0, step = v.count("step") ? atoi(v["step"].c_str()) : 0;
  if (c.empty()) return fail_usage("No contig file!", usage);
  if (b.empty()) return fail_usage("No bubble file!", usage);
  if (r.empty()) return fail_usage("No reads file!", usage);
  if (k <= 0) return fail_usage("Invalid kmer size!", usage);
  if (step <= 0 || step > 28 || step % 2 == 1) return fail_usage("Invalid step size!", usage);
  if (out.empty()) return fail_usage("No output prefix!", usage);
  o.k = (uint32_t)k;
  o.step = (uint32_t)step;
  if (k < 9 || r == "-") {  // outside the device path (k < 9; stdin): the reference's CPU path
    fprintf(stderr, "megahit_b200: iterate with k = %d is forwarded to the reference\n", k);
    // the reference's iterate refuses options it does not know: --gpus stays here
    std::vector<char *> fwd = drop_option(argc + 1, full_argv, opts, "gpus");
    return forward_to_reference(fwd.data());
  }
  // --gpus N / MHB_GPUS=N (not an option of the reference, which the Python driver never passes): one worker per GPU
  const int gpus = v.count("gpus") ? atoi(v["gpus"].c_str()) : (getenv("MHB_GPUS") ? atoi(getenv("MHB_GPUS")) : 1);
  if (int rc = gpus > 1 ? mhb_iterate_run_multi(&o, gpus) : mhb_iterate_run(&o)) {
    fprintf(stderr, "FATAL megahit_b200: %s\n", mhb_last_error());
    (void)rc;
    exit(1);
  }
  return 0;
}

// main_read2sdbg (main_sdbg_build.cpp:88-156)
int main_read2sdbg(int argc, char **argv, char **full_argv) {
  RssRecorder rec;
  const std::vector<Opt> opts = {{"kmer_k", "k", false},         {"min_kmer_frequency", "m", false}, {"host_mem", "", false},
                                 {"num_cpu_threads", "", false}, {"read_lib_file", "", false},       {"output_prefix", "", false},
                                 {"mem_flag", "", false},        {"need_mercy", "", true},           {"gpus", "", false}};
  const char *usage = "Usage: sdbg_builder read2sdbg --read_lib_file fastx_file -o out";
  std::map<std::string, std::string> v;
  std::string err;
  if (!parse(argc, argv, opts, &v, &err)) return fail_usage(err, usage);
  mhb_read2sdbg_opts o;
  memset(&o, 0, sizeof(o));
  o.k = v.count("kmer_k") ? (uint32_t)atoi(v["kmer_k"].c_str()) : 21;  // read_to_sdbg.h:36-45 defaults
  o.m = v.count("min_kmer_frequency") ? atoi(v["min_kmer_frequency"].c_str()) : 2;
  o.host_mem = v.count("host_mem") ? atof(v["host_mem"].c_str()) : 0;
  o.num_cpu_threads = v.count("num_cpu_threads") ? atoi(v["num_cpu_threads"].c_str()) : 0;
  o.mem_flag = v.count("mem_flag") ? atoi(v["mem_flag"].c_str()) : 1;
  o.need_mercy = v.count("need_mercy") ? 1 : 0;
  const std::string lib = v["read_lib_file"], out = v.count("output_prefix") ? v["output_prefix"] : "out";
  o.read_lib_file = lib.c_str();
  o.output_prefix = out.c_str();
  if (lib.empty()) return fail_usage("No input file!", usage);
  if (o.host_mem == 0) return fail_usage("Please specify the host memory!", usage);
  // --gpus N / MHB_GPUS=N (not an option of the reference, which the Python driver never passes): one worker per GPU
  const int gpus = v.count("gpus") ? atoi(v["gpus"].c_str()) : (getenv("MHB_GPUS") ? atoi(getenv("MHB_GPUS")) : 1);
  if (int rc = gpus > 1 ? mhb_read2sdbg_run_multi(&o, gpus) : mhb_read2sdbg_run(&o)) {
    fprintf(stderr, "FATAL megahit_b200: %s\n", mhb_last_error());
    (void)rc;
    exit(1);
  }
  return 0;
}

// main_build_lib (main_buildlib.cpp): the GPU path reads plain text; stdin ("-") and gzip files (a regular file whose
// first two bytes are 1f 8b, checked with pread so nothing is consumed) go to the reference, which links zlib.
bool buildlib_needs_reference(const char *lib_file) {
  std::ifstream cfg(lib_file);
  if (!cfg.is_open()) return false;  // mhb_buildlib_run reports it as the reference does
  std::string metadata, type, f1, f2;
  while (std::getline(cfg, metadata)) {
    cfg >> type;
    std::vector<std::string> files;
    if (type == "pe") {
      cfg >> f1 >> f2;
      files = {f1, f2};
    } else if (type == "se" || type == "interleaved") {
      cfg >> f1;
      files = {f1};
    } else {
      return false;
    }
    for (const auto &f : files) {
      if (f == "-") return true;
      struct stat sb;
      if (stat(f.c_str(), &sb) != 0 || !S_ISREG(sb.st_mode)) continue;
      const int fd = open(f.c_str(), O_RDONLY);
      if (fd < 0) continue;
      unsigned char m[2] = {0, 0};
      const ssize_t n = pread(fd, m, 2, 0);
      close(fd);
      if (n == 2 && m[0] == 0x1f && m[1] == 0x8b) return true;
    }
    std::getline(cfg, metadata);
  }
  return false;
}

int main_buildlib(int argc, char **argv, char **full_argv) {
  if (argc < 3) {
    fprintf(stderr, "Usage %s <read_lib_file> <out_prefix>\n", argv[0]);
    exit(1);
  }
  if (buildlib_needs_reference(argv[1])) {
    fprintf(stderr, "megahit_b200: buildlib with stdin or gzip input is forwarded to the reference\n");
    return forward_to_reference(full_argv);
  }
  RssRecorder rec;
  if (mhb_buildlib_run(argv[1], argv[2])) {
    fprintf(stderr, "FATAL %-30s: %4d - %s\n", "megahit_b200", __LINE__, mhb_last_error());
    exit(1);
  }
  return 0;
}

int forward_to_reference(char **argv) {
  std::string ref;
  if (const char *e = getenv("MHB_REFERENCE_CORE")) ref = e;
  else {
    char self[4096];
    const ssize_t n = readlink("/proc/self/exe", self, sizeof(self) - 1);
    if (n > 0) {
      self[n] = 0;
      ref = std::string(self);
      ref = ref.substr(0, ref.find_last_of('/') + 1) + "megahit_core_ref";
    }
  }
  if (ref.empty() || access(ref.c_str(), X_OK) != 0) {
    fprintf(stderr, "megahit_b200: sub-command '%s' is not part of the GPU path; set MHB_REFERENCE_CORE to the reference megahit_core to forward it\n", argv[1]);
    return 1;
  }
  argv[0] = const_cast<char *>(ref.c_str());
  execv(ref.c_str(), argv);
  perror("execv");
  return 1;
}

}  // namespace

int main(int argc, char **argv) {
  if (argc < 2) {
    fprintf(stderr, "Usage: %s <sub_program> [sub options]\n    GPU sub-programs: buildlib, count, seq2sdbg, read2sdbg, iterate; everything else is forwarded to the reference megahit_core\n", argv[0]);
    return 1;
  }
  const std::string cmd = argv[1];
  if (cmd == "count") return main_count(argc - 1, argv + 1);
  if (cmd == "seq2sdbg") return main_seq2sdbg(argc - 1, argv + 1);
  if (cmd == "read2sdbg") return main_read2sdbg(argc - 1, argv + 1, argv);
  if (cmd == "iterate") return main_iterate(argc - 1, argv + 1, argv);
  if (cmd == "buildlib") return main_buildlib(argc - 1, argv + 1, argv);
  if (cmd == "checkcpu" || cmd == "checkpopcnt" || cmd == "checkbmi2") {
    printf("1\n");
    return 0;
  }
  if (cmd == "dumpversion") {
    printf("v1.2.9\n");
    return 0;
  }
  if (cmd == "kmax") {
    printf("%d\n", MHB_MAX_K);
    return 0;
  }
  return forward_to_reference(argv);
}
