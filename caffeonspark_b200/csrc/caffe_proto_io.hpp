// caffe_proto_io.hpp -- Caffe-compatible snapshot files without libprotobuf.
//
// The reference snapshots through protobuf (solver.cpp:452-459
// SnapshotToBinaryProto -> Net::ToProto; sgd_solver.cpp:260-276
// SnapshotSolverStateToBinaryProto) and restores with
// Net::CopyTrainedLayersFrom (match layers by NAME, blobs by index and shape)
// and SGDSolver::RestoreSolverStateFromBinaryProto.  The wire subset needed is
// tiny, so it is encoded/decoded by hand (field numbers from
// caffe-public/src/caffe/proto/caffe.proto):
//   NetParameter   { name = 1; repeated LayerParameter layer = 100 }
//   LayerParameter { name = 1; type = 2; repeated BlobProto blobs = 7 }
//   BlobProto      { BlobShape shape = 7; repeated float data = 5 [packed];
//                    legacy num/channels/height/width = 1..4 (read only) }
//   BlobShape      { repeated int64 dim = 1 [packed] }
//   SolverState    { iter = 1; learned_net = 2; repeated BlobProto history = 3;
//                    current_step = 4 }
// Files written here load in stock Caffe / pycaffe; files written by Caffe for
// the same net load here.
#ifndef COS_CAFFE_PROTO_IO_HPP_
#define COS_CAFFE_PROTO_IO_HPP_

#include <cstdint>
#include <string>
#include <vector>

namespace cosb {

struct BlobView {  // one learnable blob (or one history blob) to write
  std::string layer_name;
  std::string layer_type;
  std::vector<int64_t> shape;
  const float* data = nullptr;  // host pointer, prod(shape) elements
  uint64_t count = 0;
  int param_index = -1;  // index within its layer (the HDF5 dataset name); -1: its place among the layer's views
};

struct ParsedBlob {
  std::vector<int64_t> shape;
  std::vector<float> data;
  bool present = true;  // false: an HDF5 layer group without this index's dataset (a shared param Net::ToHDF5 skips)
};

struct ParsedLayer {
  std::string name, type;
  std::vector<ParsedBlob> blobs;
};

// Consecutive BlobViews with the same layer_name form one LayerParameter.
bool write_caffemodel(const std::string& path, const std::string& net_name, const std::vector<BlobView>& blobs,
                      std::string* err);
bool read_caffemodel(const std::string& path, std::string* net_name, std::vector<ParsedLayer>* layers,
                     std::string* err);

bool write_solverstate(const std::string& path, int iter, int current_step, const std::string& learned_net,
                       const std::vector<BlobView>& history, std::string* err);

// snapshot_format: HDF5 (hdf5_io.hpp).  Same content as Net::ToHDF5 (net.cpp:867-917: /data/<layer>/<j> float
// datasets with the blob's shape) and SGDSolver::SnapshotSolverStateToHDF5 (sgd_solver.cpp:279-301: /iter,
// /learned_net, /current_step, /history/<i>).  read_caffemodel / read_solverstate recognise HDF5 files by their
// signature, so restore() works with either format (net.cpp:805-851, sgd_solver.cpp:325-347).
bool write_caffemodel_h5(const std::string& path, const std::vector<BlobView>& blobs, std::string* err);
bool write_solverstate_h5(const std::string& path, int iter, int current_step, const std::string& learned_net,
                          const std::vector<BlobView>& history, std::string* err);
bool read_solverstate(const std::string& path, int* iter, int* current_step, std::string* learned_net,
                      std::vector<ParsedBlob>* history, std::string* err);
// A file holding one BlobProto (a mean.binaryproto): shape from `shape` or the legacy num/channels/height/width.
bool read_blobproto(const std::string& path, ParsedBlob* blob, std::string* err);

}  // namespace cosb
#endif
